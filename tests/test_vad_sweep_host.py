"""Host half of the VAD sweep (diart_b200.tune.VoiceActivitySweep): the detection error oracle on exact cases and against the
DER oracle with one label per side, trial names, speech-reference packing, component arithmetic and the argument errors of
the C entry points.  No GPU needed."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks
from diart_b200.core import Annotation, Segment
from diart_b200.tune import (DetectionErrorComponents, VoiceActivitySweep, pack_speech_references, speech_reference,
                             trial_params, VAD_PARAMS)
from oracle.der import der_components
from oracle.detection import detection_components, detection_error_rate


def ann(segments, label="speech", uri="u"):
    a = Annotation(uri=uri)
    for i, (s, e) in enumerate(segments):
        a[Segment(s, e), i] = label if isinstance(label, str) else label[i]
    return a


# reference [2, 4) + [6, 8); dyadic times, so every sum is exact
EXACT = [
    ("hypothesis before the reference", [(0.0, 1.0)], [(2.0, 4.0), (6.0, 8.0)], (1.0, 4.0, 4.0)),
    ("hypothesis after the reference", [(9.0, 9.5)], [(2.0, 4.0), (6.0, 8.0)], (0.5, 4.0, 4.0)),
    ("hypothesis across the reference", [(1.0, 7.0)], [(2.0, 4.0), (6.0, 8.0)], (3.0, 1.0, 4.0)),
    ("hypothesis inside, two pieces", [(2.5, 3.0), (3.5, 6.5)], [(2.0, 4.0), (6.0, 8.0)], (2.0, 2.5, 4.0)),
    ("hypothesis equals the reference", [(2.0, 4.0), (6.0, 8.0)], [(2.0, 4.0), (6.0, 8.0)], (0.0, 0.0, 4.0)),
    ("overlapping hypothesis segments", [(1.0, 3.0), (2.0, 5.0)], [(2.0, 4.0), (6.0, 8.0)], (2.0, 2.0, 4.0)),
    ("empty hypothesis", [], [(2.0, 4.0), (6.0, 8.0)], (0.0, 4.0, 4.0)),
    ("empty reference", [(1.0, 1.5), (3.0, 5.0)], [], (2.5, 0.0, 0.0)),
    ("both empty", [], [], (0.0, 0.0, 0.0)),
]


@pytest.mark.parametrize("name,hyp,ref,want", EXACT, ids=[c[0] for c in EXACT])
def test_oracle_on_exact_cases(name, hyp, ref, want):
    got = detection_components(ann(ref), ann(hyp))
    assert got.tolist() == list(want), name


def test_oracle_merges_a_falsy_reference_gap():
    """a 1e-7 s gap between reference segments is a falsy Segment: the support merges them, nothing is missed there"""
    ref = ann([(2.0, 3.0), (3.0 + 1e-7, 4.0)], label=["a", "b"])
    comp = detection_components(ref, ann([(2.0, 4.0)]))
    assert comp.tolist() == [0.0, 0.0, 2.0]
    rows, total = speech_reference(ref)
    assert rows.tolist() == [[2.0, 4.0]] and total == 2.0
    # 1e-5 s is a real gap: two rows, and a hypothesis over it is a false alarm of that length
    ref = ann([(2.0, 3.0), (3.0 + 1e-5, 4.0)])
    rows, total = speech_reference(ref)
    assert rows.tolist() == [[2.0, 3.0], [3.0 + 1e-5, 4.0]] and total == 1.0 + (4.0 - (3.0 + 1e-5))
    fa, miss, tot = detection_components(ref, ann([(2.0, 4.0)]))
    assert fa == (3.0 + 1e-5) - 3.0 and miss == 0.0 and tot == total


def test_oracle_rate():
    assert detection_error_rate([1.0, 0.5, 6.0]) == 0.25
    assert detection_error_rate([0.0, 0.0, 0.0]) == 0.0 and detection_error_rate([0.5, 0.0, 0.0]) == 1.0


def random_side(rng, n, label_count):
    segs, labels = [], []
    t = rng.uniform(-3, 3)
    for _ in range(n):
        a = t + rng.uniform(-1.0, 4.0)
        b = a + rng.uniform(0.05, 5.0)
        segs.append((a, b))
        labels.append(f"l{rng.integers(label_count)}")
        t = a
    return segs, labels


@pytest.mark.parametrize("seed", range(40))
def test_oracle_equals_the_der_oracle_with_one_label_per_side(seed):
    """what the device computes for the VAD sweep: the DER walk with both sides collapsed to one label"""
    rng = np.random.default_rng(seed)
    rs, rl = random_side(rng, int(rng.integers(0, 12)), 3)
    hs, hl = random_side(rng, int(rng.integers(0, 12)), 2)
    ref, hyp = ann(rs, label=rl), ann(hs, label=hl)
    fa, miss, total = detection_components(ref, hyp)
    one = der_components(ann(rs), ann(hs))
    assert (fa, miss) == (one[0], one[1]), seed
    assert total == speech_reference(ref)[1]
    assert abs(total - one[4]) <= 1e-9 * max(1.0, total)    # the DER walk's total is a sum of pieces, not the durations


def test_trial_params_of_the_vad_sweep():
    cfg = blocks.VoiceActivityDetectionConfig(segmentation=object(), device=torch.device("cpu"), tau_active=0.6)
    assert VAD_PARAMS == ("tau_active",)
    p = trial_params([{}, {"tau_active": 0.25}], cfg, VAD_PARAMS)
    assert p.shape == (2, 1) and p[:, 0].tolist() == [0.6, 0.25]
    for name in ("rho_update", "delta_new", "latency", "step", "gamma"):
        with pytest.raises(ValueError, match="cannot be swept"):
            trial_params([{"tau_active": 0.5, name: 0.1}], cfg, VAD_PARAMS)
    # the default names are the diarization pipeline's, as before
    dcfg = blocks.SpeakerDiarizationConfig(segmentation=object(), embedding=object(), device=torch.device("cpu"))
    assert trial_params([{"rho_update": 0.1}], dcfg).shape == (1, 3)


def test_speech_references_pack_per_file():
    a = ann([(0.0, 2.0), (1.0, 3.0), (2.5, 4.0), (7.0, 8.0), (7.5, 7.75)], label=["x", "y", "x", "z", "x"])
    b = Annotation(uri="b")                                   # no segments: no rows, total 0
    c = ann([(5.0, 6.0), (6.0, 6.5)])                         # touching segments merge
    rows, offsets, totals = pack_speech_references([a, b, c])
    assert offsets.tolist() == [0, 2, 2, 3]
    assert rows.tolist() == [[0.0, 4.0], [7.0, 8.0], [5.0, 6.5]]
    assert totals.tolist() == [5.0, 0.0, 1.5]
    assert rows.dtype == np.float64 and rows.flags.c_contiguous and offsets.dtype == np.int32


def test_detection_error_components_arithmetic():
    a = DetectionErrorComponents(np.array([1.0, 0.0, 0.5]), np.array([0.5, 0.0, 0.0]), np.array([6.0, 0.0, 0.0]))
    b = DetectionErrorComponents(np.array([0.5, 0.0, 0.0]), np.array([1.0, 0.0, 0.0]), np.array([2.0, 0.0, 0.0]))
    assert a.detection_error_rate.tolist() == [0.25, 0.0, 1.0]
    s = a + b
    assert s.as_array().tolist() == [[1.5, 1.5, 8.0], [0.0, 0.0, 0.0], [0.5, 0.0, 0.0]]
    assert s.detection_error_rate.tolist() == [0.375, 0.0, 1.0]


def test_constructor_argument_errors_without_a_gpu():
    cfg = blocks.VoiceActivityDetectionConfig(segmentation=object(), device=torch.device("cpu"))
    with pytest.raises(ValueError):
        VoiceActivitySweep(cfg, [])
    with pytest.raises(ValueError, match="no samples"):
        VoiceActivitySweep(cfg, [("a", np.zeros(16000, np.float32), None), ("b", np.zeros(0, np.float32), None)])


def test_entry_points_reject_bad_arguments_without_a_gpu():
    lib = _lib.lib()
    ham = np.hamming(293)
    h = ctypes.c_void_p()
    for frames, k, nw, hp in ((0, 3, 1, ham), (1024, 3, 1, ham), (293, 0, 1, ham), (293, 65, 1, ham), (293, 3, 0, ham),
                              (293, 3, 257, ham), (293, 3, 1, None)):
        rc = lib.dg_vad_sweep_create(frames, k, nw, None if hp is None else hp.ctypes.data, 0, ctypes.byref(h))
        assert rc == -1 and b"dg_vad_sweep_create" in lib.dg_last_error(), (frames, k, nw)
    off = np.array([0, 1], np.int32)
    plan = np.array([[1, 29, 0, 0, 0]], np.int32)
    assert lib.dg_vad_sweep_curve(None, None, 1, 1, off.ctypes.data, plan.ctypes.data, None) == -1
    assert b"dg_vad_sweep_curve" in lib.dg_last_error()
    taus = np.array([0.5])
    n = ctypes.c_int()
    assert lib.dg_vad_sweep_run_files(None, taus.ctypes.data, 1, None, None, 0, ctypes.byref(n), None) == -1
    assert b"dg_vad_sweep_run_files" in lib.dg_last_error()
    assert lib.dg_vad_sweep_score_files(None, taus.ctypes.data, 1, None, None, None, 0.05, None, None, None, None) == -1
    assert b"dg_vad_sweep_score_files" in lib.dg_last_error()
    assert lib.dg_vad_sweep_destroy(None) == 0
