"""Host side of the multi-stream VAD server (diart_b200.serve.MultiStreamVoiceActivityDetection, dg_multi_create_vad), no GPU:
the handle's argument refusals, and the one conversion of post-path turns to VoiceActivityDetection's speech annotations."""
import ctypes as C
import math

import numpy as np
import pytest

from diart_b200 import _lib
from diart_b200.blocks.post import chunk_annotations
from diart_b200.blocks.vad import speech_annotations

HAM = np.hamming(293)
VALID = dict(chunk=80000, step=8000, streams=4, wps=4, tau=0.6, nw=4)


def create_vad(seg=None, **kw):
    a = {**VALID, **kw}
    out = C.c_void_p()
    return _lib.lib().dg_multi_create_vad(seg, a["chunk"], a["step"], a["streams"], a["wps"], a["tau"], a["nw"],
                                          HAM.ctypes.data, C.byref(out))


@pytest.mark.parametrize("kw, what", [
    (dict(), b"null handle"),
    (dict(chunk=79998), b"multiples of 4"),
    (dict(step=6), b"multiples of 4"),
    (dict(step=0), b"multiples of 4"),
    (dict(step=80004), b"step <= chunk"),
    (dict(nw=0), b"num_windows"),
    (dict(nw=257), b"num_windows"),
    (dict(tau=math.nan), b"finite threshold"),
    (dict(tau=math.inf), b"finite threshold"),
    (dict(streams=16384, wps=4), b"65535"),
    (dict(streams=0), b"max_streams"),
], ids=["null", "chunk", "step", "step0", "step_gt_chunk", "nw0", "nw257", "tau_nan", "tau_inf", "too_many_rows", "streams0"])
def test_create_vad_refusals(kw, what):
    lib = _lib.lib()
    before = lib.dg_launch_count()
    assert create_vad(**kw) == -1
    msg = lib.dg_last_error()
    assert b"dg_multi_create_vad" in msg and what in msg, msg
    assert lib.dg_launch_count() == before


def old_vad_annotations(header, turns, n, out_start, out_res, shift):
    """VoiceActivityDetection.__call__'s conversion as it read before the helper: DevicePostPath.run's annotations (one
    speaker, label speaker0), then tracks numbered in order, label "speech" """
    outputs = []
    for ann in chunk_annotations(header, turns, n, out_start, out_res, ["speaker0"], shift):
        speech = type(ann)(uri=ann.uri, modality="speech")
        for k, (segment, _) in enumerate(ann.itertracks()):
            speech[segment, k] = "speech"
        outputs.append(speech)
    return outputs


def hand_built(rng, B=6, frames=60):
    """headers {offset, count, frames, 0} with the chunks' turn blocks out of row order, and packed turns 0 << 20 | on << 10
    | off of random activity per chunk"""
    blocks, counts = [], []
    for _ in range(B):
        act = rng.random(frames) < 0.4
        act[rng.integers(0, frames):] &= rng.random() < 0.5
        edges = np.diff(np.concatenate([[0], act.astype(int), [0]]))
        on, off = np.flatnonzero(edges == 1), np.flatnonzero(edges == -1)
        blocks.append(((on << 10) | off).astype(np.uint32))
        counts.append(len(on))
    order = rng.permutation(B)
    header = np.zeros((B, 4), np.int32)
    turns, o = [], 0
    for c in order:
        header[c] = (o, counts[c], frames, 0)
        turns.append(blocks[c])
        o += counts[c]
    turns = np.concatenate(turns + [np.zeros(5, np.uint32)])
    out_start = 3.0 + 0.5 * np.arange(B)
    out_start[0] = 0.0
    out_res = np.full(B, 0.5 / frames)
    out_res[0] = 3.5 / frames
    return header, turns, o, out_start, out_res


@pytest.mark.parametrize("shift", [0.0, 2.75, "per_chunk"])
def test_speech_annotations_equal_the_former_conversion(shift):
    rng = np.random.default_rng(41)
    for _ in range(5):
        header, turns, n, out_start, out_res = hand_built(rng)
        s = np.array([0.0, 1.5, 0.0, 4.25, 2.0, 0.0]) if shift == "per_chunk" else shift
        got = speech_annotations(header, turns, n, out_start, out_res, s)
        want = old_vad_annotations(header, turns, n, out_start, out_res, s)
        assert len(got) == len(want) == len(header)
        assert sum(len(list(a.itertracks())) for a in got) == n
        for g, w in zip(got, want):
            assert (g.uri, g.modality) == (w.uri, w.modality) == (None, "speech")
            assert list(g.itertracks(yield_label=True)) == list(w.itertracks(yield_label=True))
            assert g.to_rttm() == w.to_rttm()
