"""Scoring protocols on the host: the protocol oracle (tests/scoring_protocol.py) against the collar-0 oracles and hand-built
dyadic cases, tune.scored_regions and the cropped reference packing against the oracle's steps, and the refusals of the
metric, uem and scored-region arguments without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks
from diart_b200.core import Annotation, Segment
from diart_b200.tune import (WHOLE_LINE, DetectionErrorRate, DiarizationErrorRate, VoiceActivitySweep, check_uem,
                             metric_protocol, pack_regions, reference_arrays, scored_regions, speech_reference)
from oracle import der as plain_der
from oracle import detection as plain_detection
from oracle.der import der
from oracle.detection import crop, gaps, support, timeline
from scoring_protocol import crop_annotation, der_components, detection_components, removed_regions, scored
from test_der_host import ann, brute_force_der, random_annotation

PROTOCOLS = [(0.0, False), (0.25, False), (0.5, False), (0.0, True), (0.25, True), (1.0, True)]


def random_uem(rng):
    t = np.unique(rng.integers(0, 70, 2 * int(rng.integers(1, 4)))) / 4.0 - 0.5
    return [(a, b) for a, b in zip(t[0::2], t[1::2]) if b > a] or None


def random_case(seed):
    rng = np.random.default_rng(seed)
    ref = random_annotation(rng, int(rng.integers(0, 6)), [f"spk{i}" for i in range(5)])
    hyp = random_annotation(rng, int(rng.integers(0, 6)), [f"speaker{i}" for i in range(5)])
    return rng, ref, hyp


@pytest.mark.parametrize("seed", range(30))
def test_defaults_equal_the_collar_zero_oracles_bit_for_bit(seed):
    _, ref, hyp = random_case(seed)
    hyp[Segment(0.1 + seed / 7, 0.3 + seed / 3), 99] = "speaker0"          # times that are not dyadic
    assert np.array_equal(der_components(ref, hyp), plain_der.der_components(ref, hyp))
    assert np.array_equal(detection_components(ref, hyp), plain_detection.detection_components(ref, hyp))


def comps(fa=0.0, miss=0.0, conf=0.0, corr=0.0, total=0.0):
    return np.array([fa, miss, conf, corr, total])


EPS = 2.0 ** -21      # below pyannote's 1e-6 s precision, exact in float64

# name: reference, hypothesis, (collar, skip_overlap, uem), DER components, detection components
CASES = {
    "a collar wider than a segment removes its label": (
        {"A": [(0, 4)], "B": [(6, 6.25)]}, {"x": [(0, 4)], "y": [(5, 8)]}, (1.0, False, None),
        comps(fa=1.75, corr=3, total=3), [1.75, 0.0, 3.0]),
    "skip_overlap with two labels on one segment": (
        {"A": [(0, 2)], "B": [(0, 2), (3, 4)], "C": [(3.5, 5)]}, {"x": [(0, 5)]}, (0.0, True, None),
        comps(fa=1, conf=0.5, corr=1, total=1.5), [1.0, 0.0, 1.5]),
    "a uem cutting segments of both sides": (
        {"A": [(1, 5)], "B": [(6, 9)]}, {"x": [(0, 3)], "y": [(4, 8)]}, (0.0, False, [(2, 7)]),
        comps(fa=1, miss=1, conf=1, corr=2, total=4), [1.0, 1.0, 4.0]),
    "hypothesis pieces within 1e-6 s of a scored edge are dropped": (
        {"A": [(2, 7)]}, {"x": [(0, 2 + EPS)], "y": [(3, 4)], "z": [(7 - EPS, 9)]}, (0.0, False, [(2, 7)]),
        comps(miss=4, corr=1, total=5), [0.0, 4.0, 5.0]),
    "collar, skip_overlap and a uem at once": (
        {"A": [(0, 4)], "B": [(3, 6)]}, {"x": [(0, 6)]}, (0.5, True, [(1, 5.5)]),
        comps(conf=1.25, corr=1.75, total=3), [0.0, 0.0, 3.0]),
}


@pytest.mark.parametrize("name", list(CASES))
def test_hand_built_cases(name):
    ref, hyp, (collar, skip, uem), want_der, want_det = CASES[name]
    ref, hyp = ann(ref), ann(hyp)
    got = der_components(ref, hyp, collar, skip, uem)
    assert np.array_equal(got, want_der), (got, want_der)
    speech = lambda a: ann({"speech": [(s.start, s.end) for s, _ in a.itertracks()]})   # noqa: E731
    got = detection_components(speech(ref), speech(hyp), collar, skip, uem)
    assert got.tolist() == want_det, (got, want_det)


def test_the_collar_of_the_last_case():
    # A (0, 4), B (3, 6): removed (-.25, .25) (2.75, 3.25) (3.75, 4.25) (5.75, 6.25) and the overlap (3, 4); within the uem
    # (1, 5.5) the scored regions are (1, 2.75) and (4.25, 5.5): A keeps 1.75 s, B 1.25 s, and x (mapped to A) covers both
    ref = ann({"A": [(0, 4)], "B": [(3, 6)]})
    assert scored(ref, ann({}), 0.5, True, [(1, 5.5)]) == [(1.0, 2.75), (4.25, 5.5)]


@pytest.mark.parametrize("seed", range(40))
def test_protocol_der_is_default_der_on_cropped_annotations_and_optimal(seed):
    rng, ref, hyp = random_case(seed)
    collar, skip = PROTOCOLS[seed % len(PROTOCOLS)]
    uem = random_uem(rng) if seed % 3 else None
    got = der_components(ref, hyp, collar, skip, uem)
    regions = scored_regions(ref, collar, skip, uem)          # the host's regions (whole line without a uem)
    cr, ch = crop_annotation(ref, regions), crop_annotation(hyp, regions)
    assert np.array_equal(got, plain_der.der_components(cr, ch))
    assert der(got) == brute_force_der(cr, ch)
    fa, miss, conf, corr, total = got
    assert miss + conf + corr == total


@pytest.mark.parametrize("seed", range(30))
def test_host_regions_and_cropped_references_equal_the_oracle_steps(seed):
    rng, ref, hyp = random_case(seed)
    ref[Segment(1.0, 2.0), "dup"] = "spk0"                     # a segment carried by two labels
    ref[Segment(1.0, 2.0), "dup2"] = "spk1"
    collar, skip = PROTOCOLS[seed % len(PROTOCOLS)]
    uem = random_uem(rng)
    if uem is not None:
        assert scored_regions(ref, collar, skip, uem) == scored(ref, hyp, collar, skip, uem)
    assert scored_regions(ref, collar, skip) == gaps(support(removed_regions(ref, collar, skip)), [WHOLE_LINE])
    regions = scored_regions(ref, collar, skip, uem)
    rows, labels, names = reference_arrays(ref, regions)
    want_rows, want_labels, want_names = reference_arrays(crop_annotation(ref, regions))
    assert names == want_names and np.array_equal(labels, want_labels) and np.array_equal(rows, want_rows)
    assert [[tuple(r) for r in rows[labels == k].tolist()] for k in range(len(names))] == \
        plain_der.label_unions(crop_annotation(ref, regions))
    srows, total = speech_reference(ref, regions)
    want = support(crop(timeline(ref), regions))
    assert [tuple(r) for r in srows.tolist()] == want
    assert total == detection_components(ref, crop_annotation(ref, regions), collar, skip, regions)[2]
    # without regions the packing is what it was
    assert np.array_equal(reference_arrays(ref)[0], reference_arrays(ref, None)[0])


def test_metric_and_uem_refusals():
    assert metric_protocol(None, "DiarizationErrorRate") == (0.0, False)
    assert metric_protocol(DiarizationErrorRate(0.25, True), "DiarizationErrorRate") == (0.25, True)
    assert metric_protocol(DetectionErrorRate(collar=1), "DetectionErrorRate") == (1.0, False)

    class DiarizationErrorRateLike:                     # pyannote's own class is accepted by name
        collar, skip_overlap = 0.5, False
    DiarizationErrorRateLike.__name__ = "DiarizationErrorRate"
    assert metric_protocol(DiarizationErrorRateLike(), "DiarizationErrorRate") == (0.5, False)
    for bad in (DetectionErrorRate(), "DiarizationErrorRate", object(), DiarizationErrorRate(-0.1),
                DiarizationErrorRate(float("nan")), DiarizationErrorRate(float("inf")), DiarizationErrorRate("0.25")):
        with pytest.raises(ValueError):
            metric_protocol(bad, "DiarizationErrorRate")
    assert check_uem([Segment(0, 1), (2, 3.5)]) == [(0.0, 1.0), (2.0, 3.5)]
    for bad in ((0, 1), [(1, 1 + 1e-7)], [(2, 3), (0, 1)], [(0, float("nan"))], [(1, 0)], "0 1", [(0, 1, 2)]):
        with pytest.raises(ValueError):
            check_uem(bad)
    with pytest.raises(ValueError):
        scored_regions(ann({"A": [(0, 1)]}), -0.5)
    cfg = blocks.VoiceActivityDetectionConfig(segmentation=object(), device=torch.device("cpu"))
    x = np.zeros(16000, np.float32)
    with pytest.raises(ValueError, match="uems"):
        VoiceActivitySweep(cfg, [("a", x, None), ("b", x, None)], uems=[None])
    with pytest.raises(ValueError, match="falsy"):
        VoiceActivitySweep(cfg, [("a", x, None)], uems=[[(0.0, 1e-7)]])


def test_scored_region_setters_refuse_without_a_gpu():
    lib = _lib.lib()
    for name in ("dg_sweep_set_scored_regions", "dg_vad_sweep_set_scored_regions"):
        setter = getattr(lib, name)
        good = pack_regions([[(0.0, 1.0), (2.0, 3.0)], []])
        bad_rows = {
            "overlap": np.array([[0.0, 2.0], [1.0, 3.0]]),
            "apart by 1e-6 s or less": np.array([[0.0, 1.0], [1.0 + 5e-7, 3.0]]),
            "not sorted": np.array([[2.0, 3.0], [0.0, 1.0]]),
            "falsy": np.array([[0.0, 5e-7], [2.0, 3.0]]),
            "nan": np.array([[0.0, np.nan], [2.0, 3.0]]),
            "infinite": np.array([[-np.inf, 1.0], [2.0, 3.0]]),
        }
        for what, rows in bad_rows.items():
            rows = np.ascontiguousarray(rows)
            assert setter(None, 2, rows.ctypes.data, good[1].ctypes.data) == -1, what
            assert name.encode() in lib.dg_last_error() and b"null handle" not in lib.dg_last_error(), what
        for off in (np.array([1, 2, 2], np.int32), np.array([0, 2, 1], np.int32)):
            assert setter(None, 2, good[0].ctypes.data, off.ctypes.data) == -1
        assert setter(None, -1, None, None) == -1
        assert setter(None, 1, good[0].ctypes.data, None) == -1
        assert setter(None, 2, good[0].ctypes.data, good[1].ctypes.data) == -1
        assert b"null handle" in lib.dg_last_error()
