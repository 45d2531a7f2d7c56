"""Diarization and detection error rate components under a scoring protocol -- a forgiveness collar, ``skip_overlap`` and a
uem -- restated from pyannote.metrics' ``uemify`` (test infrastructure: the device scorers with scored regions are compared
against it bit for bit).  Definition in DESIGN.md "DER scoring", steps 1-5.

The steps run literally, per (reference, hypothesis) pair, in Python floats, with the pyannote.core restatements of
``oracle/detection.py`` (``support``, ``crop``, ``gaps``, ``co_iter``):

  1. uem        the given one, else the extent of the reference's timeline ``|`` the hypothesis's
  2. removed    around both ends of every unique non-empty reference segment ``Segment(t - .5 * collar, t + .5 * collar)``
                (collar > 0); with ``skip_overlap`` the intersection of every pair of ``reference.co_iter(reference)`` but
                a track with itself
  3. scored     ``Timeline(removed).support().gaps(support=uem)``
  4. crop       both annotations, every segment cut against each scored piece it intersects, falsy pieces dropped
  5. score      ``oracle.der.der_components`` on the cropped annotations; detection error as ``oracle.detection`` with the
                scored pieces as the uem

With the defaults (collar 0, no skip_overlap, no uem) steps 2-4 are the identity and both functions return the bits of
``oracle.der.der_components`` / ``oracle.detection.detection_components``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from diart_b200.core import Annotation, Segment
from oracle import der as _der
from oracle.detection import (Seg, co_iter, crop, duration, extent, gaps, intersection, intersects, support, timeline, truthy,
                              union)


def all_pairs(segs: List[Seg]):
    """``Timeline.co_iter`` of a sorted timeline with itself, literally: every y not after (x.end, x.end) is tested"""
    for x in segs:
        for y in segs:
            if y > (x[1], x[1]):
                break
            if intersects(x, y):
                yield x, y


def removed_regions(reference: Annotation, collar: float = 0.0, skip_overlap: bool = False) -> List[Seg]:
    """step 2, the truthy removed regions in the order pyannote appends them"""
    tracks = {}
    for s, t in reference.itertracks():
        if s:
            tracks.setdefault((s.start, s.end), []).append(t)
    segs = sorted(tracks)
    removed: List[Seg] = []
    if collar > 0.0:
        for s, e in segs:
            for t in (s, e):
                removed.append((t - .5 * collar, t + .5 * collar))
    if skip_overlap:
        for x, y in all_pairs(segs):
            for t1 in sorted(tracks[x], key=str):
                for t2 in sorted(tracks[y], key=str):
                    if (x, t1) != (y, t2):
                        removed.append(intersection(x, y))
    return [r for r in removed if truthy(r)]


def uem_of(reference: Annotation, hypothesis: Annotation, uem: Optional[Sequence] = None) -> List[Seg]:
    """step 1"""
    if uem is not None:
        return [p for p in ((float(a), float(b)) for a, b in uem) if truthy(p)]
    u = union(extent(timeline(reference)), extent(timeline(hypothesis)))
    return [u] if truthy(u) else []


def scored(reference: Annotation, hypothesis: Annotation, collar: float = 0.0, skip_overlap: bool = False,
           uem: Optional[Sequence] = None) -> List[Seg]:
    """steps 1-3"""
    return gaps(support(removed_regions(reference, collar, skip_overlap)), uem_of(reference, hypothesis, uem))


def crop_annotation(annotation: Annotation, regions: List[Seg]) -> Annotation:
    """step 4: ``annotation.crop(regions, mode="intersection")`` (an Annotation keeps no falsy segment)"""
    labels = {}
    for s, _, label in annotation.itertracks(yield_label=True):
        if s:
            labels.setdefault((s.start, s.end), []).append(label)
    out = Annotation(uri=annotation.uri, modality=annotation.modality)
    n = 0
    for x, r in co_iter(sorted(labels), regions):
        p = intersection(x, r)
        if truthy(p):
            for label in labels[x]:
                out[Segment(*p), n] = label
                n += 1
    return out


def der_components(reference: Annotation, hypothesis: Annotation, collar: float = 0.0, skip_overlap: bool = False,
                   uem: Optional[Sequence] = None) -> np.ndarray:
    """float64 (5,) = false alarm, missed detection, confusion, correct, total of ``DiarizationErrorRate(collar,
    skip_overlap)(reference, hypothesis, uem=uem)``'s components"""
    regions = scored(reference, hypothesis, collar, skip_overlap, uem)
    return _der.der_components(crop_annotation(reference, regions), crop_annotation(hypothesis, regions))


def detection_components(reference: Annotation, hypothesis: Annotation, collar: float = 0.0, skip_overlap: bool = False,
                         uem: Optional[Sequence] = None) -> np.ndarray:
    """float64 (3,) = false alarm, missed detection, total of ``DetectionErrorRate(collar, skip_overlap)``: both sides
    cropped to the scored pieces, then their supports, gaps per scored piece and the sums of ``oracle.detection``"""
    regions = scored(reference, hypothesis, collar, skip_overlap, uem)
    ref, hyp = support(crop(timeline(reference), regions)), support(crop(timeline(hypothesis), regions))
    ref_gaps, hyp_gaps = gaps(ref, regions), gaps(hyp, regions)
    false_alarm = 0.0
    for r_, h in co_iter(ref_gaps, hyp):
        false_alarm += duration(intersection(r_, h))
    miss = 0.0
    for r, h_ in co_iter(ref, hyp_gaps):
        miss += duration(intersection(r, h_))
    total = 0.0
    for r in ref:
        total += duration(r)
    return np.array([false_alarm, miss, total], dtype=np.float64)
