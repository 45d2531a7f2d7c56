"""Host half of per-stream latency and thresholds in the multi-stream servers (diart_b200/serve.py), without a GPU: the plan of
a tick whose streams are at several latencies, and the argument checks that refuse a stream before the handle is touched."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks, models
from diart_b200.blocks.aggregation import DelayedAggregation
from diart_b200.serve import (MultiStreamDiarization, MultiStreamVoiceActivityDetection, _MultiStreamServer, mixed_plan,
                              plan_rows, stream_windows)

SR, S, HOP, F = 16000, 80000, 8000, 293


def tick_rows(rng, latencies, max_wps=4):
    """the rows of a tick of streams at `latencies`, each at its own position, grouped by stream -> (stream of each row,
    chunk index of each row)"""
    stream, idx = [], []
    for k in range(len(latencies)):
        first, n = int(rng.integers(0, 40)), int(rng.integers(1, max_wps + 1))
        stream += [k] * n
        idx += list(range(first, first + n))
    return np.array(stream), np.array(idx)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_mixed_latency_plan_equals_plan_rows_per_stream(seed):
    rng = np.random.default_rng(seed)
    latencies = [0.5, 1.0, 2.0, 5.0, 1.5, 0.5, 5.0, 3.0]
    nw_max = stream_windows(5.0, 0.5)
    stream, idx = tick_rows(rng, latencies)
    res = np.where(stream % 3 == 0, 1 / SR, (220500 / 44100) / S)          # a few rows of resampled streams
    lat = np.array(latencies)[stream]
    plan, out_start, out_res = mixed_plan(idx, lat, 0.5, S, SR, F, nw_max, res)
    assert plan.shape == (len(idx), 4 + nw_max) and plan.dtype == np.int32
    for r in range(len(idx)):
        nw = stream_windows(lat[r], 0.5)
        want, s, o = plan_rows(idx[r:r + 1], 0.5, S, SR, F, nw, float(lat[r]), res[r:r + 1])
        assert np.array_equal(plan[r, :4 + nw], want[0]), f"row {r}"
        assert not plan[r, 4 + nw:].any(), f"row {r}: the tail beyond the stream's buffers is not 0"
        assert plan[r, 0] <= nw
        assert out_start[r] == s[0] and out_res[r] == o[0], f"row {r}"


def test_one_latency_is_the_plan_of_today():
    """every stream at the server's largest latency: the one plan_rows evaluation of a server without per-stream latency"""
    idx = np.concatenate([np.arange(0, 4), np.arange(37, 40), np.arange(116, 120)])
    for latency in (0.5, 2.0, 5.0):
        nw = stream_windows(latency, 0.5)
        got = mixed_plan(idx, np.full(len(idx), latency), 0.5, S, SR, F, nw, 1 / SR)
        want = plan_rows(idx, 0.5, S, SR, F, nw, latency, np.full(len(idx), 1 / SR))
        for g, w in zip(got, want):
            assert g.dtype == w.dtype and np.array_equal(g, w)
    empty = mixed_plan(np.zeros(0, np.int64), np.zeros(0), 0.5, S, SR, F, 4, np.zeros(0))
    assert empty[0].shape == (0, 8)


def test_stream_windows_is_delayed_aggregation():
    for latency in (0.5, 0.75, 1.0, 1.26, 2.0, 4.9, 5.0):
        assert stream_windows(latency, 0.5) == DelayedAggregation(0.5, latency).num_overlapping_windows


def fake_server(latency=2.0, max_latency=5.0):
    cfg = types.SimpleNamespace(sample_rate=SR, step=0.5, duration=5.0, latency=latency, tau_active=0.6, rho_update=0.3,
                                delta_new=1.0)
    fake = types.SimpleNamespace(config=cfg, max_latency=max_latency, rates={SR: (-1, S, HOP, 1 / SR)}, _resamplers={},
                                 _open=np.zeros(2, bool))
    return fake


@pytest.mark.parametrize("kw, what", [
    (dict(latency=0.25), "latency"),
    (dict(latency=5.5), "latency"),
    (dict(tau_active=math.nan), "tau_active"),
    (dict(rho_update=math.inf), "rho_update"),
    (dict(delta_new=-math.inf), "delta_new"),
    (dict(sample_rate=44100), "sample rate"),
], ids=["below_step", "above_max", "tau_nan", "rho_inf", "delta_ninf", "rate"])
def test_open_refusals_before_the_handle(kw, what):
    """a refused open raises ValueError before any call into the library (the fake server has no handle)"""
    fake = fake_server()
    with pytest.raises(ValueError, match=what):
        MultiStreamDiarization.open(fake, **kw)
    assert not fake._open.any()


def test_vad_open_takes_latency_and_tau_only():
    fake = fake_server()
    for kw in (dict(rho_update=0.3), dict(delta_new=1.0)):
        with pytest.raises(TypeError):
            MultiStreamVoiceActivityDetection.open(fake, **kw)
    with pytest.raises(ValueError, match="tau_active"):
        MultiStreamVoiceActivityDetection.open(fake, tau_active=math.nan)
    with pytest.raises(ValueError, match="latency"):
        MultiStreamVoiceActivityDetection.open(fake, latency=0.1)


@pytest.mark.parametrize("max_latency", [1.5, 5.5])
def test_max_latency_outside_the_config_range_is_refused(max_latency):
    """max_latency below the config's latency or above its duration: refused before a model is touched"""
    foreign = models.SegmentationModel(lambda: torch.nn.Identity())
    vad = blocks.VoiceActivityDetectionConfig(segmentation=foreign, latency=2.0, device=torch.device("cpu"))
    with pytest.raises(ValueError, match="max_latency"):
        MultiStreamVoiceActivityDetection(vad, 2, max_latency=max_latency)
    dia = types.SimpleNamespace(step=0.5, duration=5.0, latency=2.0, max_speakers=4)
    with pytest.raises(ValueError, match="max_latency"):
        _MultiStreamServer.__init__(types.SimpleNamespace(), dia, 2, 4, (), (), max_latency)


def test_open_config_refuses_a_null_handle():
    lib = _lib.lib()
    params = np.array([0.5, 0.3, 1.0])
    before = lib.dg_launch_count()
    assert lib.dg_multi_open_config(None, 0, -1, 1, params.ctypes.data) == -1
    assert b"dg_multi_open_config" in lib.dg_last_error()
    assert lib.dg_launch_count() == before
