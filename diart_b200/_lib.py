"""ctypes binding of libdiartb200.so (include/diart_b200.h).

There is deliberately NO fallback: if the shared library cannot be loaded, or no CUDA device is
present when a compute entry point is called, the caller gets an exception.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdiartb200.so")

_lib: Optional[C.CDLL] = None


class DgTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("numel", C.c_int64)]


# name -> (restype, argtypes); mirrors include/diart_b200.h one to one
_P = C.c_void_p
SIGNATURES = {
    "dg_last_error": (C.c_char_p, []),
    "dg_version": (C.c_int, []),
    "dg_launch_count": (C.c_int64, []),
    "dg_profile_enable": (C.c_int, [C.c_int]),
    "dg_profile_report": (C.c_int, [C.c_char_p, C.c_int]),
    "dg_selftest_gemm_tc": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float),
                                      C.POINTER(C.c_float)]),
    "dg_selftest_gemm_tc_grid": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "dg_selftest_gemm_tc_bounds": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                             C.POINTER(C.c_int)]),
    "dg_selftest_wgmma_row_shift": (C.c_int, [C.c_int, C.POINTER(C.c_uint)]),
    "dg_selftest_wgmma_b_row_shift": (C.c_int, [C.c_int, C.POINTER(C.c_uint)]),
    "dg_selftest_gemm_tc_pool3_simt": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float),
                                                 C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "dg_selftest_gemm_tc_halo": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int),
                                           C.POINTER(C.c_int)]),
    "dg_selftest_split_f16_host": (C.c_int, [_P, C.c_longlong, _P, _P]),
    "dg_seg_create": (C.c_int, [C.POINTER(DgTensor), C.c_int, C.c_int, C.POINTER(_P)]),
    "dg_seg_dims": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "dg_seg_set_powerset": (C.c_int, [_P, C.c_int, C.c_int]),
    "dg_seg_forward": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P]),
    "dg_seg_destroy": (C.c_int, [_P]),
    "dg_emb_create": (C.c_int, [C.POINTER(DgTensor), C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "dg_emb_dims": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "dg_emb_forward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P]),
    "dg_emb_forward_rows": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "dg_emb_destroy": (C.c_int, [_P]),
    "dg_emb_debug_trunk": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int64, _P]),
    "dg_seg_debug_stage": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int64, _P]),
    "dg_emb_debug_stage": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int64, _P]),
    "dg_selftest_sinc_filters_host": (C.c_int, [_P, _P, _P]),
    "dg_selftest_fbank_tables_host": (C.c_int, [_P, _P]),
    "dg_osp": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, _P, _P]),
    "dg_normalize_embeddings": (C.c_int, [_P, C.c_int, C.c_int, C.c_float, _P, _P]),
    "dg_cluster_create": (C.c_int, [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.POINTER(_P)]),
    "dg_cluster_set_metric": (C.c_int, [_P, C.c_int]),
    "dg_cluster_step": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "dg_cluster_reset": (C.c_int, [_P]),
    "dg_cluster_get_state": (C.c_int, [_P, _P, _P, C.POINTER(C.c_int)]),
    "dg_cluster_set_state": (C.c_int, [_P, _P, _P, C.c_int]),
    "dg_cluster_destroy": (C.c_int, [_P]),
    "dg_cluster_record_len": (C.c_int, [_P]),
    "dg_cluster_export_delta": (C.c_int, [_P, _P, _P]),
    "dg_cluster_merge": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int, _P]),
    "dg_pipeline_identity_export": (C.c_int, [_P, _P, _P]),
    "dg_pipeline_identity_merge": (C.c_int, [_P, _P, C.c_int, C.c_int, _P]),
    "dg_pipeline_create": (C.c_int, [_P, _P, _P, C.c_float, C.c_float, C.c_int, C.POINTER(_P)]),
    "dg_pipeline_set_hop": (C.c_int, [_P, C.c_int]),
    "dg_pipeline_step": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "dg_pipeline_step_host": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, _P, _P]),
    "dg_pipeline_submit": (C.c_int, [_P, _P, C.c_int, C.c_int, _P]),
    "dg_pipeline_collect": (C.c_int, [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), _P]),
    "dg_pipeline_collect_copy": (C.c_int, [_P, _P, _P, _P, _P]),
    "dg_pipeline_submit_host": (C.c_int, [_P, _P, C.c_int, C.c_int]),
    "dg_pipeline_collect_host": (C.c_int, [_P, _P, _P, _P]),
    "dg_pipeline_destroy": (C.c_int, [_P]),
    "dg_pipeline_nets_sets": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, C.c_int64, _P]),
    "dg_post_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_double, C.c_int, C.POINTER(_P)]),
    "dg_post_step": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.POINTER(C.c_int), _P]),
    "dg_post_reset": (C.c_int, [_P]),
    "dg_post_destroy": (C.c_int, [_P]),
    "dg_stream_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "dg_stream_push_host": (C.c_int, [_P, _P, C.c_int]),
    "dg_stream_available": (C.c_int, [_P]),
    "dg_stream_windows": (C.c_int, [_P, C.c_int, _P, _P]),
    "dg_stream_reset": (C.c_int, [_P]),
    "dg_stream_destroy": (C.c_int, [_P]),
    "dg_pipeline_submit_stream": (C.c_int, [_P, _P, C.c_int]),
    "dg_pipeline_call_stream": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.POINTER(C.c_int), _P, _P]),
    "dg_pipeline_call_host": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int, C.POINTER(C.c_int), _P, _P]),
    "dg_pipeline_last_call_h2d_bytes": (C.c_int64, [_P]),
    "dg_resample_create": (C.c_int, [C.c_int, C.c_int, _P, C.c_int, C.c_int, C.POINTER(_P)]),
    "dg_resample_out_len": (C.c_int64, [_P, C.c_int64]),
    "dg_resample_forward": (C.c_int, [_P, _P, C.c_int, C.c_int64, _P, _P]),
    "dg_resample_destroy": (C.c_int, [_P]),
    "dg_stream_create_resampled": (C.c_int, [C.c_int, C.c_int, _P, C.c_int, C.c_int, C.POINTER(_P)]),
    "dg_stream_crop_host": (C.c_int, [_P, C.c_int, _P, _P]),
    "dg_sweep_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, C.POINTER(_P)]),
    "dg_sweep_run": (C.c_int, [_P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, C.c_int, C.POINTER(C.c_int), _P]),
    "dg_sweep_destroy": (C.c_int, [_P]),
    "dg_sweep_set_scored_regions": (C.c_int, [_P, C.c_int, _P, _P]),
    "dg_sweep_set_trial_sets": (C.c_int, [_P, C.c_int, _P, C.c_int]),
    "dg_sweep_set_seeds": (C.c_int, [_P, C.c_int, _P, _P]),
    "dg_sweep_set_identities": (C.c_int, [_P, C.c_int, _P]),
    "dg_sweep_score": (C.c_int, [_P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, C.c_double, C.c_double, _P, _P, C.c_int,
                                 C.c_int, _P, _P, _P, C.c_int, _P]),
    "dg_sweep_run_files": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, _P, _P, _P, _P, _P, C.c_int,
                                     C.POINTER(C.c_int), _P]),
    "dg_sweep_score_files": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int, _P, _P, _P, _P, C.c_double, _P, _P,
                                       _P, _P, _P, _P, _P, C.c_int, _P]),
    "dg_sweep_state_order": (C.c_int, [C.c_int, _P, C.c_int, _P]),
    "dg_sweep_run_latencies": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int, _P, _P,
                                         _P, _P, C.c_int, C.POINTER(C.c_int), _P]),
    "dg_sweep_score_latencies": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int, _P, _P,
                                           _P, _P, C.c_double, _P, _P, _P, _P, _P, _P]),
    "dg_sweep_check_latencies": (C.c_int, [C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int, C.c_int]),
    "dg_vad_sweep_curve_latencies": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, _P]),
    "dg_vad_sweep_create": (C.c_int, [C.c_int, C.c_int, C.c_int, _P, C.c_int, C.POINTER(_P)]),
    "dg_vad_sweep_curve": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "dg_vad_sweep_run_files": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_int, C.POINTER(C.c_int), _P]),
    "dg_vad_sweep_score_files": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, C.c_double, _P, _P, _P, _P]),
    "dg_vad_sweep_destroy": (C.c_int, [_P]),
    "dg_vad_sweep_set_scored_regions": (C.c_int, [_P, C.c_int, _P, _P]),
    "dg_multi_create": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double,
                                  C.c_float, C.c_float, C.c_int, C.c_int, _P, C.POINTER(_P)]),
    "dg_multi_create_vad": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, _P, C.POINTER(_P)]),
    "dg_multi_open": (C.c_int, [_P, C.c_int]),
    "dg_multi_close": (C.c_int, [_P, C.c_int]),
    "dg_multi_push_host": (C.c_int, [_P, C.c_int, _P, C.c_int]),
    "dg_multi_available": (C.c_int, [_P, C.c_int]),
    "dg_multi_step": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, C.c_int, C.POINTER(C.c_int), _P, _P, _P]),
    "dg_multi_last_step_ms": (C.c_int, [_P, C.POINTER(C.c_float)]),
    "dg_multi_destroy": (C.c_int, [_P]),
    "dg_selftest_multi_staging_host": (C.c_int, [C.c_int, C.c_int, C.c_int, _P, _P, _P, _P]),
    "dg_multi_add_rate": (C.c_int, [_P, _P, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "dg_multi_open_rate": (C.c_int, [_P, C.c_int, C.c_int]),
    "dg_multi_open_config": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "dg_multi_open_seeded": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, _P, C.c_int]),
    "dg_multi_get_state": (C.c_int, [_P, C.c_int, _P, _P, C.POINTER(C.c_int)]),
    "dg_multi_last_windows": (C.c_int, [_P, _P, C.c_int]),
    "dg_gallery_create": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "dg_gallery_destroy": (C.c_int, [_P]),
    "dg_gallery_query": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_double, _P, _P, _P]),
    "dg_multi_set_gallery": (C.c_int, [_P, _P, C.c_double]),
    "dg_multi_set_names": (C.c_int, [_P, C.c_int, C.c_uint32, _P]),
    "dg_multi_set_slot_gallery": (C.c_int, [_P, C.c_int, _P, C.c_double]),
    "dg_selftest_gallery_plan_host": (C.c_int, [C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, C.c_int, _P]),
    "dg_selftest_multi_gallery_host": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, C.c_char_p,
                                                 C.c_int]),
    "dg_multi_last_names": (C.c_int, [_P, _P, C.c_int, C.POINTER(C.c_int)]),
    "dg_selftest_multi_frames_host": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P, C.c_int,
                                                C.POINTER(C.c_int)]),
    "dg_multi_export_bytes": (C.c_int, [_P, _P, C.c_int, _P]),
    "dg_multi_export": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int64]),
    "dg_multi_import": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P]),
    "dg_selftest_multi_transfer_host": (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int64, _P,
                                                  C.c_char_p, C.c_int]),
}


class DiartB200Error(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Loads (building first if the sources are newer and nvcc exists) libdiartb200.so."""
    global _lib
    if _lib is not None:
        return _lib
    from . import build as _build

    if not os.path.exists(LIB_PATH) or (_build._stale() and _build.have_nvcc()):
        _build.build()
    try:
        handle = C.CDLL(LIB_PATH)
    except OSError as e:  # loud: no eager / CPU fallback exists
        raise DiartB200Error(f"cannot load {LIB_PATH}: {e}. Run `python -m diart_b200.build`.") from e
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = res, args
    _lib = handle
    return handle


def check(rc: int):
    """Maps status codes to the exception types the reference raises for the same misuse."""
    if rc == 0:
        return
    msg = lib().dg_last_error().decode()
    if rc == -1:
        if "Cannot update unknown centers" in msg:
            raise AssertionError(msg)
        raise ValueError(msg)
    if rc == -3:
        raise KeyError(msg)
    raise DiartB200Error(f"libdiartb200 error {rc}: {msg}")


def require_cuda(device: torch.device):
    if device.type != "cuda":
        raise DiartB200Error(
            f"diart_b200 runs on CUDA devices only (got '{device}'); there is no CPU implementation")
    if not torch.cuda.is_available():
        raise DiartB200Error("diart_b200 needs a CUDA device (sm_90a); none is available")


def pack_state_dict(state: Dict[str, "torch.Tensor | np.ndarray"]):
    """state_dict -> (ctypes array of dg_tensor, keep-alive list)."""
    keep, items = [], []
    for name, value in state.items():
        arr = value.detach().cpu().numpy() if isinstance(value, torch.Tensor) else np.asarray(value)
        if arr.dtype.kind != "f":
            continue  # e.g. BatchNorm num_batches_tracked
        arr = np.ascontiguousarray(arr, dtype=np.float32)
        bname = name.encode()
        keep.extend([arr, bname])
        items.append(DgTensor(bname, arr.ctypes.data, arr.size))
    array = (DgTensor * len(items))(*items)
    keep.append(array)
    return array, len(items), keep


def stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()
