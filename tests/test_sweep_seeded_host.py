"""Seeded sweeps and the identification error rate without a GPU: the IER oracle on hand-built cases and against DER on
random ones, the name -> hypothesis label table the host builds for dg_sweep_set_identities, per-file speaker labels in
the assembled predictions, the metric checks, and the null-handle refusals of the two setters."""
import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from diart_b200 import _lib
from diart_b200.core import Annotation, Segment
from diart_b200.speakers import KnownSpeakers, speaker_labels
from diart_b200.tune import (DatasetSweep, DiarizationErrorRate, IdentificationErrorComponents, IdentificationErrorRate,
                             SweepOutputs, diarization_metric, identity_table, metric_protocol, pack_identities,
                             reference_arrays, scored_regions)
from ier_oracle import ier_components, named_unions, protocol_ier_components
from oracle.der import activity, der, der_components
from scoring_protocol import crop_annotation, der_components as protocol_der_components, scored
from test_der_host import ann, comps
from test_scoring_protocol_host import PROTOCOLS, random_uem

CASES = {
    "names right": ({"alice": [(0, 2)], "bob": [(1, 3)]}, {"alice": [(0, 2)], "bob": [(1, 3)]}, comps(corr=4, total=4), 0.0),
    "names swapped": ({"alice": [(0, 2)], "bob": [(1, 3)]}, {"bob": [(0, 2)], "alice": [(1, 3)]},
                      comps(conf=2, corr=2, total=4), 0.5),
    "unknown names": ({"alice": [(0, 2)]}, {"speaker0": [(0, 2)]}, comps(conf=2, total=2), 1.0),
    "one name right, one absent": ({"alice": [(0, 1)], "bob": [(1, 3)]}, {"alice": [(0, 1)], "speaker1": [(1, 3)]},
                                   comps(conf=2, corr=1, total=3), 2 / 3),
    "false alarm and miss": ({"alice": [(0, 1)], "bob": [(2, 3)]}, {"alice": [(0, 1.5)]},
                             comps(fa=0.5, miss=1, corr=1, total=2), 0.75),
    "empty hypothesis": ({"alice": [(0, 1.5)]}, {}, comps(miss=1.5, total=1.5), 1.0),
    "empty reference": ({}, {"alice": [(0, 1)]}, comps(fa=1), 1.0),
    "both empty": ({}, {}, comps(), 0.0),
}


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_hand_built_cases(name):
    ref, hyp, want, want_ier = CASES[name]
    got = ier_components(ann(ref), ann(hyp))
    assert np.array_equal(got, want), (got, want)
    assert der(got) == want_ier
    assert IdentificationErrorComponents.from_array(got[None]).ier[0] == want_ier


def der_mapping(ref: Annotation, hyp: Annotation):
    """{hypothesis name: reference name} of the oracle's optimal mapping (linear_sum_assignment on the co-occurrence)"""
    rn, ru = named_unions(ref)
    hn, hu = named_unions(hyp)
    bounds = np.unique(np.array([t for u in ru + hu for seg in u for t in seg], dtype=np.float64))
    lo, hi = bounds[:-1], bounds[1:]
    keep = np.array([bool(Segment(a, b)) for a, b in zip(lo.tolist(), hi.tolist())], dtype=bool)
    lo, hi = lo[keep], hi[keep]
    d = hi - lo
    if not (rn and hn and len(d)):
        return {}
    ar, ah = activity(ru, lo, hi), activity(hu, lo, hi)
    C = np.cumsum(np.where(ar[:, None, :] & ah[None, :, :], d[None, None, :], 0.0), axis=2)[:, :, -1]
    rows, cols = linear_sum_assignment(-C)
    return {hn[h]: rn[r] for r, h in zip(rows, cols)}


def renamed(hyp: Annotation, mapping) -> Annotation:
    """the hypothesis with every mapped label renamed to its reference label, the others to names no reference has"""
    out = Annotation(uri=hyp.uri)
    for n, (s, _, label) in enumerate(hyp.itertracks(yield_label=True)):
        out[s, n] = mapping.get(label, f"unmapped-{label}")
    return out


def seeded_case(seed):
    """up to 5 labels per side with dyadic times; the hypothesis draws its names from the reference's, speaker<g> and
    names the reference lacks"""
    rng = np.random.default_rng(seed)
    pool = [f"spk{i}" for i in range(5)] + [f"speaker{i}" for i in range(3)] + ["zed"]
    ref = random_annotation(rng, int(rng.integers(0, 6)), [f"spk{i}" for i in range(5)])
    hyp = random_annotation(rng, int(rng.integers(0, 6)), list(rng.permutation(pool)[:5]))
    return rng, ref, hyp


def random_annotation(rng, n_labels, names):
    spec = {}
    for k in range(n_labels):
        n = rng.integers(1, 5)
        t = np.sort(rng.integers(0, 64, 2 * n)) / 4.0        # quarter seconds: every sum is exact
        spec[names[k]] = [(a, b) for a, b in zip(t[0::2], t[1::2]) if b > a]
    return ann(spec)


@pytest.mark.parametrize("seed", range(40))
def test_ier_against_der_on_seeded_cases(seed):
    rng, ref, hyp = seeded_case(seed)
    got_ier, got_der = ier_components(ref, hyp), der_components(ref, hyp)
    assert der(got_ier) >= der(got_der)
    assert np.array_equal(got_ier[[0, 1, 4]], got_der[[0, 1, 4]])     # only the matching differs
    # IER on the hypothesis renamed by DER's mapping is DER, bit for bit
    assert np.array_equal(ier_components(ref, renamed(hyp, der_mapping(ref, hyp))), got_der)
    # the protocol: IER on the annotations cropped to the scored regions
    collar, skip = PROTOCOLS[seed % len(PROTOCOLS)]
    uem = random_uem(rng)
    regions = scored(ref, hyp, collar, skip, uem)
    want = ier_components(crop_annotation(ref, regions), crop_annotation(hyp, regions))
    assert np.array_equal(protocol_ier_components(ref, hyp, collar, skip, uem), want)
    assert der(protocol_ier_components(ref, hyp, collar, skip, uem)) >= der(protocol_der_components(ref, hyp, collar,
                                                                                                      skip, uem))
    assert np.array_equal(protocol_ier_components(ref, hyp), got_ier)


def test_identity_table():
    labels = speaker_labels(KnownSpeakers(["alice", "bob"], np.eye(2, 4)), 5)
    assert labels == ["alice", "bob", "speaker2", "speaker3", "speaker4"]
    # reference names in string order: bob, carol (reference only), speaker3, speaker9 (no such speaker)
    ref = ann({"speaker3": [(0, 1)], "carol": [(1, 2)], "bob": [(2, 3)], "speaker9": [(3, 4)]})
    names = reference_arrays(ref)[2]
    assert names == ["bob", "carol", "speaker3", "speaker9"]
    table = identity_table(names, labels)
    assert table.dtype == np.int32 and table.shape == (32,)
    assert table[:4].tolist() == [1, -1, 3, -1] and (table[4:] == -1).all()   # alice (hypothesis only) is nobody's
    # an unseeded file's labels are speaker<g>
    assert identity_table(names, speaker_labels(None, 5))[:4].tolist() == [-1, -1, 3, -1]
    # per file, after cropping: a label left without a piece disappears from the names
    regions = [[(2.5, 3.5)], None]
    packed = pack_identities([ref, ref], regions, [labels, speaker_labels(None, 5)])
    assert packed.shape == (2, 32) and packed.flags.c_contiguous
    assert packed[0, :2].tolist() == [1, -1] and (packed[0, 2:] == -1).all()
    assert packed[1, :4].tolist() == [-1, -1, 3, -1]


def test_predictions_carry_each_files_labels():
    """DatasetSweep._run assembles file f's turns with labels[f]: speaker 0 of chunk 0 (file 0) and of chunk 1 (file 1)"""
    ds = object.__new__(DatasetSweep)
    ds.uris, ds.offsets = ["a", "b"], np.array([0, 1, 2], dtype=np.int32)
    ds.out_start, ds.out_res, ds.shifts = np.zeros(2), np.full(2, 0.1), np.zeros(2)
    ds.timing = {}
    header = np.array([[[0, 2, 0, 0], [2, 1, 0, 0]]], dtype=np.int32)
    turns = np.array([(0 << 20) | (0 << 10) | 5, (1 << 20) | (2 << 10) | 8, (0 << 20) | (1 << 10) | 4], dtype=np.uint32)
    out = SweepOutputs(header, turns, 3, ds.out_start, ds.out_res)
    labels = [speaker_labels(KnownSpeakers(["alice"], np.ones((1, 3))), 3), speaker_labels(None, 3)]
    runs = ds._run(np.zeros((1, 3)), lambda _: out, labels)
    assert sorted(runs[0][0].labels()) == ["alice", "speaker1"]
    assert runs[1][0].labels() == ["speaker0"]


class IdentificationErrorRateLike:
    """pyannote.metrics' class, as far as the sweep reads it"""

    def __init__(self, collar=0.0, skip_overlap=False, confusion=1.0, miss=1.0, false_alarm=1.0):
        self.collar, self.skip_overlap = collar, skip_overlap
        self.confusion, self.miss, self.false_alarm = confusion, miss, false_alarm


IdentificationErrorRateLike.__name__ = "IdentificationErrorRate"


def test_metric_acceptance_and_refusals():
    assert diarization_metric(None) == ("DiarizationErrorRate", 0.0, False)
    assert diarization_metric(DiarizationErrorRate(0.5, True)) == ("DiarizationErrorRate", 0.5, True)
    assert diarization_metric(IdentificationErrorRate()) == ("IdentificationErrorRate", 0.0, False)
    assert diarization_metric(IdentificationErrorRate(collar=0.25, skip_overlap=True)) == \
        ("IdentificationErrorRate", 0.25, True)
    assert diarization_metric(IdentificationErrorRateLike(0.25, False, 1, 1.0, np.float64(1))) == \
        ("IdentificationErrorRate", 0.25, False)
    for kw in ({"confusion": 0.5}, {"miss": 2.0}, {"false_alarm": 0.0}, {"miss": True}, {"confusion": "1"}):
        name = next(iter(kw))
        with pytest.raises(ValueError, match=f"metric {name} weight"):
            diarization_metric(IdentificationErrorRateLike(**kw))
    with pytest.raises(ValueError, match="collar"):
        diarization_metric(IdentificationErrorRate(collar=-1.0))
    with pytest.raises(ValueError, match="scores a DiarizationErrorRate"):
        diarization_metric(object())
    # the single-file sweep and the VAD sweep keep refusing it
    with pytest.raises(ValueError, match="scores a DiarizationErrorRate"):
        metric_protocol(IdentificationErrorRate(), "DiarizationErrorRate")
    with pytest.raises(ValueError, match="scores a DetectionErrorRate"):
        metric_protocol(IdentificationErrorRate(), "DetectionErrorRate")
    assert scored_regions(ann({"a": [(0, 1)]}), *diarization_metric(IdentificationErrorRate(0.5))[1:]) == \
        scored_regions(ann({"a": [(0, 1)]}), 0.5)


def test_components_type():
    a = IdentificationErrorComponents.from_array(np.array([[1.0, 2.0, 3.0, 4.0, 9.0], [0.0, 0.0, 0.0, 1.0, 1.0]]))
    b = IdentificationErrorComponents.from_array(np.array([[0.0, 0.0, 0.0, 1.0, 1.0], [1.0, 0.0, 0.0, 0.0, 0.0]]))
    s = a + b
    assert isinstance(s, IdentificationErrorComponents)
    assert np.array_equal(s.as_array(), a.as_array() + b.as_array())
    assert np.array_equal(s.ier, [0.6, 1.0])


def test_setters_refuse_a_null_handle():
    lib = _lib.lib()
    off = np.array([0, 1], dtype=np.int32)
    centers = np.ones((1, 4))
    table = np.full((1, 32), -1, dtype=np.int32)
    assert lib.dg_sweep_set_seeds(None, 1, off.ctypes.data, centers.ctypes.data) == -1
    assert b"null handle" in lib.dg_last_error()
    assert lib.dg_sweep_set_seeds(None, 0, None, None) == -1
    assert lib.dg_sweep_set_identities(None, 1, table.ctypes.data) == -1
    assert b"null handle" in lib.dg_last_error()
    assert lib.dg_sweep_set_identities(None, 0, None) == -1
