"""Host half of the hyper-parameter sweep (diart_b200/tune.py) and the argument checks of dg_sweep_create: no GPU needed."""
import ctypes
import types

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks
from diart_b200.blocks.post import DevicePostPath, post_plan
from diart_b200.sinks import PredictionAccumulator
from diart_b200.tune import assemble_predictions, file_windows, trial_params


def config(**kw):
    return blocks.SpeakerDiarizationConfig(segmentation=object(), embedding=object(), device=torch.device("cpu"), **kw)


def reference_windows(x, cfg):
    """numpy restatement of FileAudioSource.read (reference sources.py:88-127) + rearrange_audio_stream
    (operators.py:44-100): (windows, start times)"""
    sr = cfg.sample_rate
    left, right = cfg.get_file_padding(file_duration=len(x) / sr)
    w = x[None, :].astype(np.float64)
    if left > 0:
        w = np.concatenate([np.zeros((1, int(np.rint(left * sr)))), w], axis=1)
    if right > 0:
        w = np.concatenate([w, np.zeros((1, int(np.rint(right * sr))))], axis=1)
    block = int(np.rint(cfg.step * sr))
    n_full = w.shape[1] // block
    blocks_ = [w[:, i * block:(i + 1) * block] for i in range(n_full)]
    if w.shape[1] % block:
        last = w[:, n_full * block:]
        blocks_.append(np.concatenate([last, np.zeros((1, block - last.shape[1]))], axis=1))
    chunk_samples, step_samples = int(round(sr * cfg.duration)), int(round(sr * cfg.step))
    chunk, buffer, start_time, out = None, None, 0, []
    for value in blocks_:
        buffer = value if buffer is None else np.concatenate([buffer, value], axis=1)
        if buffer.shape[1] >= step_samples:
            if buffer.shape[1] == step_samples:
                new_chunk, buffer = buffer, None
            else:
                new_chunk, buffer = buffer[:, :step_samples], buffer[:, step_samples:]
            if chunk is not None:
                new_chunk = np.concatenate([chunk, new_chunk], axis=1)
            if new_chunk.shape[1] > chunk_samples:
                new_chunk = new_chunk[:, -chunk_samples:]
                start_time += cfg.step
            chunk = new_chunk
            if chunk.shape[1] == chunk_samples:
                out.append((chunk[0].copy(), start_time))
    return out, (left, right)


@pytest.mark.parametrize("kw,seconds", [({}, 7.0), ({}, 7.0 + 123 / 16000), ({}, 2.3), ({"latency": 2.0}, 9.71),
                                        ({"step": 0.3}, 8.0), ({"step": 0.3, "latency": 1.2}, 6.05)])
def test_windows_and_padding_follow_the_file_source(kw, seconds):
    cfg = config(**kw)
    x = np.random.default_rng(3).standard_normal(int(round(seconds * 16000))).astype(np.float32)
    want, padding = reference_windows(x, cfg)
    fw = file_windows(x, cfg)
    assert fw.padding == padding
    assert fw.num_windows == len(want) > 0
    for i, (w, start) in enumerate(want):
        assert np.array_equal(fw.window(i), w.astype(np.float32)), f"window {i}"
        assert fw.starts[i] == start, f"start of window {i}"


def test_trials_take_config_values_and_reject_other_keys():
    cfg = config(tau_active=0.55, rho_update=0.25, delta_new=0.9)
    p = trial_params([{}, {"tau_active": 0.7}, {"rho_update": 1, "delta_new": 0.1}], cfg)
    assert p.dtype == np.float64
    assert p.tolist() == [[0.55, 0.25, 0.9], [0.7, 0.25, 0.9], [0.55, 1.0, 0.1]]
    for bad in ({"gamma": 2.0}, {"tau_active": 0.5, "latency": 1.0}, {"max_speakers": 4}, {"tau": 0.5}):
        with pytest.raises(ValueError):
            trial_params([{}, bad], cfg)
    with pytest.raises(ValueError):
        trial_params([], cfg)


def _synthetic_turns(rng, T, N, M, F, nfo):
    """packed turns of T trials over N chunks, blocks in a shuffled order (as the device's atomic counter leaves them)"""
    per = {}
    for t in range(T):
        for c in range(N):
            turns = []
            for g in sorted(rng.choice(M, size=rng.integers(0, 4), replace=False)):
                f = int(rng.integers(0, 3))
                while f < nfo[c] - 1:
                    on = f
                    off = min(nfo[c], on + int(rng.integers(1, 8)))
                    turns.append((g << 20) | (on << 10) | off)
                    f = off + int(rng.choice([1, 2, 3, 4, 9]))       # gaps of 1-4 frames straddle the 0.05 s collar
            if t == 0 and c < N - 1 and nfo[c] > 2:                   # a turn running to the chunk's end, another from
                turns.append((M - 1 << 20) | (nfo[c] - 2 << 10) | nfo[c])  # the next chunk's first frame: they abut
                per.setdefault((t, c + 1, "head"), []).append((M - 1 << 20) | (0 << 10) | 2)
            per[(t, c)] = turns
    header = np.zeros((T, N, 4), np.int32)
    flat, order = [], rng.permutation(T * N)
    for r in order:
        t, c = divmod(int(r), N)
        turns = per[(t, c)] + per.get((t, c, "head"), [])
        turns.sort(key=lambda p: (p >> 20, (p >> 10) & 1023))
        header[t, c] = (len(flat), len(turns), nfo[c], 0)
        flat += turns
    return header, np.array(flat, dtype=np.uint32)


@pytest.mark.parametrize("latency,shift,seed", [(0.5, 0.0, 1), (2.0, -1.5, 2), (1.5, -0.25, 3)])
def test_vectorised_assembly_equals_prediction_accumulator(latency, shift, seed):
    rng = np.random.default_rng(seed)
    T, N, M, F, step = 3, 14, 20, 293, 0.5
    nw = int(round(latency / step))
    res = 5.0 / F
    starts = np.arange(N) * step
    plan, out_start, out_res = post_plan(starts, res, np.zeros(0), np.zeros(0), nw, F, step, latency)
    nfo = np.where(plan[:, 2] > 0, plan[:, 2], plan[:, 1])
    assert plan[0, 2] > 0                                         # the first chunk carries the prepended crop
    header, turns = _synthetic_turns(rng, T, N, M, F, nfo)
    labels = [f"speaker{g}" for g in range(M)]
    got = assemble_predictions(header, turns, len(turns), out_start, out_res, labels, shift, uri="file")
    host = types.SimpleNamespace(labels=labels)                  # DevicePostPath.annotations only reads the labels
    lines = 0
    for t in range(T):
        acc = PredictionAccumulator("file")
        own = np.concatenate([turns[o:o + n] for o, n in header[t, :, :2]])     # this trial's turns alone, chunk order
        h = header[t].copy()
        h[:, 0] = np.concatenate([[0], np.cumsum(h[:-1, 1])])
        for ann in DevicePostPath.annotations(host, h, own, len(own), out_start, out_res, shift):
            acc.on_next(ann)
        want = acc.get_prediction().to_rttm()
        assert got[t].to_rttm() == want, f"trial {t}"
        lines += want.count("\n")
    assert lines > 3 * T


def test_assembly_of_trials_without_turns():
    starts = np.arange(5) * 0.5
    plan, out_start, out_res = post_plan(starts, 5.0 / 293, np.zeros(0), np.zeros(0), 1, 293, 0.5, 0.5)
    header = np.zeros((2, 5, 4), np.int32)
    got = assemble_predictions(header, np.zeros(0, np.uint32), 0, out_start, out_res, ["speaker0", "speaker1"], uri="f")
    assert [a.to_rttm() for a in got] == ["", ""]


def test_sweep_create_rejects_out_of_range_arguments_without_a_gpu():
    lib = _lib.lib()
    ham = np.hamming(293)
    out = ctypes.c_void_p()
    for M, D, F, K, nw in ((33, 512, 293, 3, 1), (20, 512, 293, 9, 1), (20, 512, 1024, 3, 1), (20, 512, 293, 3, 0),
                           (2, 512, 293, 3, 1), (20, 512, 293, 3, 257), (20, 0, 293, 3, 1)):
        assert lib.dg_sweep_create(M, D, F, K, nw, ham.ctypes.data, 0, ctypes.byref(out)) == -1, (M, D, F, K, nw)
        assert b"dg_sweep_create" in lib.dg_last_error()
        assert out.value is None
    assert lib.dg_sweep_create(20, 512, 293, 3, 1, None, 0, ctypes.byref(out)) == -1
