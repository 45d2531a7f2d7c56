"""Gallery naming without a GPU: the float64 oracle of the naming rule (tests/gallery_oracle.py) on hand-made cases,
SpeakerGallery's checks, and the C entry points' refusals."""
import ctypes as C
import math
import types

import numpy as np
import pytest

from diart_b200 import _lib
from diart_b200.serve import MultiStreamVoiceActivityDetection
from diart_b200.speakers import KnownSpeakers, SpeakerGallery, check_gallery
from gallery_oracle import cosine_distances, first_copies, name_step, nearest, resolve

SQ = math.sqrt(0.5)


def unit(*angles_deg):
    return np.array([[math.cos(math.radians(a)), math.sin(math.radians(a))] for a in angles_deg])


def test_the_distance_is_the_clipped_cosine_distance():
    x = np.array([[1.0, 0.0], [3.0, 4.0]])
    e = np.array([[0.0, 2.0], [-1.0, 0.0], [6.0, 8.0]])
    d = cosine_distances(x, e)
    assert d[0, 0] == 1.0 and d[0, 1] == 2.0 and abs(d[1, 2]) < 1e-15 and d[1, 2] >= 0.0
    assert np.allclose(d[1], [1 - 0.8, 1 + 0.6, 0.0])


def test_a_distance_equal_to_the_threshold_names_nothing():
    names, entries = ["alice"], np.array([[0.0, 1.0]])
    centroid = np.array([[5.0, 0.0]])                 # distance exactly 1.0
    assert name_step(["speaker0"], centroid, names, entries, 1.0)[0] == ["speaker0"]
    assert name_step(["speaker0"], centroid, names, entries, np.nextafter(1.0, 2.0))[0] == ["alice"]
    assert resolve(np.array([0]), np.array([0.5]), 0.5).tolist() == [-1]


def test_duplicate_entries_go_to_the_lowest_index():
    entries = np.concatenate([unit(90, 10), unit(10, 10)])   # rows 1, 2, 3 are one direction
    assert first_copies(entries).tolist() == [0, 1, 1, 1]
    d = cosine_distances(unit(12), entries)
    assert d[0, 1] == d[0, 2] == d[0, 3]
    entry, best, runner = nearest(d)
    assert entry.tolist() == [1] and runner[0] > best[0]
    assert nearest(d, claimed=[1])[0].tolist() == [2]
    labels, _ = name_step(["speaker0"], unit(12), ["a", "b", "c", "d"], entries, 0.5)
    assert labels == ["b"]


def test_the_closer_speaker_wins_and_the_other_is_named_at_the_next_tick():
    names, entries = ["alice", "bob"], unit(0, 40)
    centroids = unit(2, 15)                 # both nearest alice; speaker 1 is 25 degrees from bob
    labels, compared = name_step(["speaker0", "speaker1"], centroids, names, entries, 0.2)
    assert labels == ["alice", "speaker1"] and len(compared) == 2
    labels, compared = name_step(labels, centroids, names, entries, 0.2)
    assert labels == ["alice", "bob"] and [c[0] for c in compared] == [1]
    # equal distances: the lower speaker wins
    labels, _ = name_step(["speaker0", "speaker1"], unit(5, -5), names[:1], entries[:1], 0.2)
    assert labels == ["alice", "speaker1"]


def test_claimed_entries_are_skipped():
    entry, best, _ = nearest(cosine_distances(unit(1), unit(0, 30, 60)), claimed=[0])
    assert entry.tolist() == [1] and abs(best[0] - (1 - math.cos(math.radians(29)))) < 1e-15
    entry, best, _ = nearest(cosine_distances(unit(1), unit(0)), claimed=[0])
    assert entry.tolist() == [-1] and best[0] == np.inf


def test_seeded_names_are_claimed_from_the_start():
    names, entries = ["alice", "bob"], unit(0, 50)
    # speaker 0 is a known "alice": speaker 1, nearest alice, cannot take her entry and gets nothing under 0.2
    labels, _ = name_step(["alice", "speaker1"], unit(0, 3), names, entries, 0.2)
    assert labels == ["alice", "speaker1"]
    # a known speaker whose name is not in the gallery claims nothing
    labels, _ = name_step(["carol", "speaker1"], unit(0, 3), names, entries, 0.2)
    assert labels == ["carol", "alice"]
    # nothing to compare once every speaker is named
    assert name_step(["carol", "alice"], unit(0, 3), names, entries, 0.2) == (["carol", "alice"], [])


def gallery(n=3, d=4, threshold=0.5, names=None):
    rng = np.random.default_rng(n)
    return SpeakerGallery(KnownSpeakers(names or [f"p{i}" for i in range(n)], rng.standard_normal((n, d))), threshold,
                          device="cuda")


def test_gallery_refusals():
    with pytest.raises(ValueError, match="label of a discovered speaker"):
        gallery(names=["p0", "speaker1", "p2"])
    with pytest.raises(ValueError, match="label of a discovered speaker"):
        gallery(names=["speaker0", "p1", "p2"])
    with pytest.raises(ValueError, match="given twice"):
        gallery(names=["p0", "p1", "p0"])
    for t in (0.0, -0.1, 2.5, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="threshold"):
            gallery(threshold=t)
    assert gallery(threshold=2.0).threshold == 2.0
    with pytest.raises(TypeError):
        SpeakerGallery(np.zeros((2, 4)), 0.5)
    g = gallery()
    with pytest.raises(ValueError, match="shape"):
        g.identify(np.ones((2, 5)))
    with pytest.raises(ValueError, match="dimension"):
        g.name(KnownSpeakers(["speaker0"], np.ones((1, 5))))
    with pytest.raises(ValueError, match="claimed"):
        g.identify(np.ones((1, 4)), claimed=[3])
    with pytest.raises(ValueError, match="metric"):
        check_gallery(g, types.SimpleNamespace(metric="euclidean"), 4)
    with pytest.raises(ValueError, match="dimension"):
        check_gallery(g, types.SimpleNamespace(), 512)
    check_gallery(g, types.SimpleNamespace(metric="cosine"), 4)
    with pytest.raises(ValueError, match="no speakers to name"):
        MultiStreamVoiceActivityDetection(None, 4, gallery=g)


def test_claims_of_a_label_list():
    g = gallery(names=["alice", "bob", "carol"])
    named, claimed = g.claims(["speaker0", "bob", "dan", "speaker3"])
    assert named == 0b0110 and claimed.tolist() == [-1, 1, -1, -1]


def test_c_entry_points_refuse_bad_arguments_without_a_device():
    lib = _lib.lib()
    out = C.c_void_p()
    good = np.ones((4, 8))
    assert lib.dg_gallery_create(None, 4, 8, 0, C.byref(out)) == -1
    for G, D in ((0, 8), ((1 << 20) + 1, 8), (4, 7), (4, 0)):
        assert lib.dg_gallery_create(good.ctypes.data, G, D, 0, C.byref(out)) == -1
        assert b"dg_gallery_create" in lib.dg_last_error()
    bad = good.copy()
    bad[2, 3] = np.nan
    assert lib.dg_gallery_create(bad.ctypes.data, 4, 8, 0, C.byref(out)) == -1 and b"entry 2" in lib.dg_last_error()
    bad = good.copy()
    bad[1] = 0.0
    assert lib.dg_gallery_create(bad.ctypes.data, 4, 8, 0, C.byref(out)) == -1 and b"zero norm" in lib.dg_last_error()
    assert lib.dg_gallery_query(None, None, 1, None, None, 0.5, None, None, None) == -1
    assert lib.dg_gallery_destroy(None) == 0
    assert lib.dg_multi_set_gallery(None, None, 0.5) == -1
    assert lib.dg_multi_set_names(None, 0, 0, None) == -1
    n = C.c_int()
    assert lib.dg_multi_last_names(None, None, 0, C.byref(n)) == -1
