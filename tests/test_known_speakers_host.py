"""Known speakers without a GPU (diart_b200.speakers): the checks of KnownSpeakers, the dominance rule of enroll, the
per-stream label lists of the annotations, and the seeding contract on the float64 oracle of the clustering -- a
clustering whose state is filled from an earlier run's state continues that run exactly."""
import numpy as np
import pytest

from diart_b200.blocks.post import chunk_annotations
from diart_b200.core import Annotation, Segment
from diart_b200.speakers import KnownSpeakers, dominant_speaker, exported, speaker_labels
from oracle.clustering import OracleClustering
from oracle.synth_cluster import make_stream
from oracle.vs_reference_inputs import CLUSTER_CONFIGS

D = 8


def unit(i, d=D):
    v = np.zeros(d)
    v[i % d] = 1.0
    return v


@pytest.mark.parametrize("names, centroids, match", [
    (["alice", "bob"], np.ones((3, D)), "2 names and 3 centroids"),
    (["alice", ""], np.ones((2, D)), "speaker 1: the name must be a non-empty string"),
    (["alice", 7], np.ones((2, D)), "speaker 1: the name must be a non-empty string"),
    (["alice", "bob smith"], np.ones((2, D)), "speaker 1: the name 'bob smith' contains whitespace"),
    (["alice\t", "bob"], np.ones((2, D)), "speaker 0: the name 'alice\\\\t' contains whitespace"),
    (["alice", "bob", "alice"], np.ones((3, D)), "speaker 2: the name 'alice' is given twice"),
    (["alice", "speaker0"], np.ones((2, D)), "speaker 1: the name 'speaker0' may only be given to speaker 0"),
    (["speaker3"], np.ones((1, D)), "speaker 0: the name 'speaker3' may only be given to speaker 3"),
    (["alice", "bob"], np.array([np.ones(D), np.r_[np.ones(D - 1), np.nan]]), r"speaker 1 \(bob\): the centroid is not "),
    (["alice", "bob"], np.array([np.r_[np.inf, np.ones(D - 1)], np.ones(D)]), r"speaker 0 \(alice\): the centroid is not "),
    (["alice", "bob"], np.array([np.ones(D), np.zeros(D)]), r"speaker 1 \(bob\): the centroid has a zero norm"),
    (["alice"], np.ones(D), r"centroids must have shape \(n, D\)"),
])
def test_refusals_name_the_entry(names, centroids, match):
    with pytest.raises(ValueError, match=match):
        KnownSpeakers(names, centroids)


def test_a_valid_construction_is_owned_and_immutable():
    c = np.stack([unit(0), unit(1), -unit(2)])
    known = KnownSpeakers(["alice", "speaker1", "Bob-2"], c)
    assert known.names == ("alice", "speaker1", "Bob-2") and len(known) == 3 and known.dimension == D
    assert known.centroids.dtype == np.float64 and known.centroids.flags.c_contiguous
    assert not known.centroids.flags.writeable
    c[0, 0] = 5.0                                      # the caller's array is not shared
    assert known.centroids[0, 0] == 1.0
    with pytest.raises(AttributeError):
        known.names = ("x",)
    with pytest.raises(ValueError):
        known.centroids[0, 0] = 2.0
    assert known == KnownSpeakers(["alice", "speaker1", "Bob-2"], np.stack([unit(0), unit(1), -unit(2)]))
    assert known != KnownSpeakers(["alice", "speaker1", "Bob-3"], np.stack([unit(0), unit(1), -unit(2)]))
    # "speaker01" and "speakerX" are not labels the clustering gives, so they may sit anywhere
    KnownSpeakers(["speaker01", "speakerX"], np.ones((2, D)))


def test_no_known_speakers():
    for empty in (KnownSpeakers([], []), KnownSpeakers((), np.zeros((0, D)))):
        assert len(empty) == 0
    assert speaker_labels(KnownSpeakers([], []), 3) == speaker_labels(None, 3) == ["speaker0", "speaker1", "speaker2"]


def test_labels_name_the_known_speakers_first():
    known = KnownSpeakers(["alice", "bob"], np.ones((2, D)))
    assert speaker_labels(known, 4) == ["alice", "bob", "speaker2", "speaker3"]
    # what a stream exports resumes with the same labels: discovered speakers come back as speaker<g> at index g
    again = exported(speaker_labels(known, 4), np.arange(4 * D, dtype=np.float64).reshape(4, D) + 1, [1, 1, 1, 0])
    assert again.names == ("alice", "bob", "speaker2")
    assert speaker_labels(again, 4) == speaker_labels(known, 4)
    with pytest.raises(AssertionError):
        exported(speaker_labels(None, 4), np.ones((4, D)), [1, 0, 1, 0])


def annotation(turns):
    ann = Annotation(uri="clip")
    for i, (a, b, label) in enumerate(turns):
        ann[Segment(a, b), i] = label
    return ann


def test_the_dominant_speaker_has_the_most_speech():
    labels = speaker_labels(None, 4)
    assert dominant_speaker(annotation([(0, 1, "speaker0"), (1, 3.5, "speaker2"), (4, 5, "speaker0")]), labels) == 2
    assert dominant_speaker(annotation([(0, 1, "speaker1"), (2, 3.5, "speaker3"), (4, 5, "speaker1")]), labels) == 1
    # a tie goes to the lowest index, whatever the order of the turns
    assert dominant_speaker(annotation([(0, 2, "speaker3"), (2, 3, "speaker1"), (5, 6, "speaker1")]), labels) == 1
    assert dominant_speaker(annotation([(0, 2, "speaker1"), (2, 4, "speaker3")]), labels) == 1
    assert dominant_speaker(annotation([]), labels) is None


def packed(g, on, off):
    return (g << 20) | (on << 10) | off


def test_annotations_take_a_label_list_per_chunk():
    """chunk_annotations with one label list per chunk: each chunk's speakers carry the labels of its own stream; with one
    shared list it builds what it always built"""
    header = np.array([[0, 2, 0, 0], [2, 1, 0, 0], [3, 2, 0, 0]], dtype=np.int32)
    turns = np.array([packed(0, 0, 3), packed(1, 2, 5), packed(0, 1, 4), packed(1, 0, 2), packed(2, 3, 6)], dtype=np.uint32)
    out_start, out_res = np.array([0.0, 0.5, 1.0]), np.full(3, 0.1)
    shared = speaker_labels(None, 3)
    seeded = speaker_labels(KnownSpeakers(["alice", "bob"], np.ones((2, D))), 3)
    plain = chunk_annotations(header, turns, 5, out_start, out_res, shared, 0.0)
    mixed = chunk_annotations(header, turns, 5, out_start, out_res, [shared, seeded, seeded], 0.0)
    same = chunk_annotations(header, turns, 5, out_start, out_res, [shared] * 3, 0.0)
    assert [a.to_rttm() for a in same] == [a.to_rttm() for a in plain]
    assert mixed[0].to_rttm() == plain[0].to_rttm()
    assert sorted(mixed[1].labels()) == ["alice"]
    assert sorted(mixed[2].labels()) == ["bob", "speaker2"]
    assert sorted(plain[2].labels()) == ["speaker1", "speaker2"]
    for a, b in zip(mixed[1:], plain[1:]):
        assert [s for s, _ in a.itertracks()] == [s for s, _ in b.itertracks()]


def replay(clu, seg, emb):
    return np.stack([clu(s, e)[0] for s, e in zip(seg, emb)])


def seeded_oracle(M, tau, rho, delta, known):
    """an OracleClustering whose public state is filled from ``known``, as set_known_speakers / open(speakers=) fill the
    device state"""
    clu = OracleClustering(tau, rho, delta, "cosine", M)
    if len(known):
        clu.centers = np.zeros((M, known.dimension))
        clu.centers[:len(known)] = known.centroids
        clu.active_centers = set(range(len(known)))
    return clu


@pytest.mark.parametrize("case", range(len(CLUSTER_CONFIGS)))
@pytest.mark.parametrize("k", [1, 9, 60])
def test_a_seeded_clustering_continues_the_run_it_was_exported_from(case, k):
    M, sigma, delta, tau, rho = CLUSTER_CONFIGS[case]
    seg, emb = make_stream(120, 300 + case, sigma=sigma)
    whole = OracleClustering(tau, rho, delta, "cosine", M)
    first = replay(whole, seg[:k], emb[:k])
    labels = speaker_labels(None, M)
    known = exported(labels, whole.centers, [int(g in whole.active_centers) for g in range(M)])
    assert len(known) > 0
    rest = replay(whole, seg[k:], emb[k:])
    resumed = seeded_oracle(M, tau, rho, delta, known)
    assert np.array_equal(replay(resumed, seg[k:], emb[k:]), rest)
    assert np.array_equal(resumed.centers.view(np.int64), whole.centers.view(np.int64))
    assert resumed.active_centers == whole.active_centers
    assert first.shape == (k, 3)


def test_an_empty_seed_is_the_fresh_state_and_an_initialised_empty_state_is_not():
    M, sigma, delta, tau, rho = CLUSTER_CONFIGS[0]
    seg, emb = make_stream(40, 77, sigma=sigma)
    seg[0, :, 2] = 0.05
    seg[0, 100:110, 2] = 0.9                          # speaker 2 of chunk 0 is active but short (mean < rho)
    fresh = replay(OracleClustering(tau, rho, delta, "cosine", M), seg, emb)
    empty = replay(seeded_oracle(M, tau, rho, delta, KnownSpeakers([], [])), seg, emb)
    assert np.array_equal(empty, fresh)
    # initialised with no active centre: the distance path from the first chunk on, which creates centres for long
    # speakers only, where the first-chunk path creates one for every active speaker
    initialised = OracleClustering(tau, rho, delta, "cosine", M)
    initialised.centers = np.zeros((M, emb.shape[2]))
    got = replay(initialised, seg, emb)
    assert fresh[0, 2] >= 0 and got[0, 2] == -1
