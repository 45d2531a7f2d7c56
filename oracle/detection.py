"""Detection error rate components, restated from pyannote.metrics' ``DetectionErrorRate(collar=0, skip_overlap=False)``
without a uem (test infrastructure: the device scorer of the VAD sweep, dg_vad_sweep_score_files, is compared against it
bit for bit).  Definition in DESIGN.md "Detection error".

Step by step as pyannote computes it, in Python floats (the same float64 operations in the same order):

  uem         ``reference extent | hypothesis extent`` (``Segment.__or__``: an empty side gives the other's extent)
  both sides  cropped to the uem (``mode="intersection"``), then ``get_timeline().support()``: segments in (start, end)
              order, a segment merged into the current one when ``Segment(current end, its start)`` is falsy
  gaps        of each side within the uem, the falsy ones dropped
  false alarm ``sum (r_ & h).duration`` over ``reference_gaps.co_iter(hypothesis)``, in that order
  miss        ``sum (r & h_).duration`` over ``reference.co_iter(hypothesis_gaps)``
  total       ``reference.duration()``: the support's durations summed in order
"""
from __future__ import annotations

import bisect
from typing import List, Optional, Tuple

import numpy as np

from diart_b200.core import Annotation

PRECISION = 1e-6      # pyannote.core SEGMENT_PRECISION

Seg = Tuple[float, float]


def truthy(s: Seg) -> bool:
    """``Segment.__bool__``"""
    return (s[1] - s[0]) > PRECISION


def duration(s: Seg) -> float:
    """``Segment.duration``: 0 for a falsy segment"""
    return s[1] - s[0] if truthy(s) else 0.0


def intersection(a: Seg, b: Seg) -> Seg:
    """``Segment.__and__``"""
    return (max(a[0], b[0]), min(a[1], b[1]))


def intersects(a: Seg, b: Seg) -> bool:
    """``Segment.intersects``"""
    return ((a[0] < b[0] and b[0] < a[1] - PRECISION) or (a[0] > b[0] and a[0] < b[1] - PRECISION)
            or a[0] == b[0])


def extent(segs: List[Seg]) -> Seg:
    """``Timeline.extent()``: first and last boundary, (0, 0) for an empty timeline"""
    if not segs:
        return (0.0, 0.0)
    return (min(s[0] for s in segs), max(s[1] for s in segs))


def union(a: Seg, b: Seg) -> Seg:
    """``Segment.__or__``"""
    if not truthy(a):
        return b
    if not truthy(b):
        return a
    return (min(a[0], b[0]), max(a[1], b[1]))


def support(segs: List[Seg]) -> List[Seg]:
    """``Timeline.support()`` (collar 0) of the unique segments in (start, end) order"""
    out: List[Seg] = []
    cur: Optional[Seg] = None
    for s in sorted(set(segs)):
        if cur is None:
            cur = s
            continue
        gap = (min(s[1], cur[1]), max(s[0], cur[0]))          # Segment.__xor__
        if not truthy(gap):
            cur = union(cur, s)
        else:
            out.append(cur)
            cur = s
    if cur is not None:
        out.append(cur)
    return out


def co_iter(a: List[Seg], b: List[Seg]):
    """``Timeline.co_iter``: pairs (x, y), x of a in order, y of b in order among those not after (x.end, x.end), that
    intersect.  ``b`` is sorted with non-decreasing ends (a support, gaps or one segment), so the y that end before x
    starts, which cannot intersect it, are skipped by bisection."""
    ends = [y[1] for y in b]
    assert all(p <= q for p, q in zip(ends, ends[1:]))
    for x in a:
        for y in b[bisect.bisect_left(ends, x[0]):]:
            if y > (x[1], x[1]):
                break
            if intersects(x, y):
                yield x, y


def crop(segs: List[Seg], uem: List[Seg]) -> List[Seg]:
    """``Timeline.crop(uem, mode="intersection")`` followed by dropping falsy pieces (an Annotation keeps no empty segment)"""
    return [p for p in (intersection(x, y) for x, y in co_iter(sorted(set(segs)), uem)) if truthy(p)]


def gaps(segs: List[Seg], uem: List[Seg]) -> List[Seg]:
    """``Timeline.gaps(support=uem)``: per uem segment, the truthy gaps between the support of the segments inside it"""
    out: List[Seg] = []
    for u in support(uem):
        end = u[0]
        for s in support(crop(segs, [u])):
            if truthy((end, s[0])):
                out.append((end, s[0]))
            end = s[1]
        if truthy((end, u[1])):
            out.append((end, u[1]))
    return out


def timeline(annotation: Annotation) -> List[Seg]:
    return [(s.start, s.end) for s, _ in annotation.itertracks() if s]


def detection_components(reference: Annotation, hypothesis: Annotation) -> np.ndarray:
    """float64 (3,) = false alarm, missed detection, total (seconds)"""
    ref, hyp = timeline(reference), timeline(hypothesis)
    u = union(extent(ref), extent(hyp))
    uem = [u] if truthy(u) else []
    ref, hyp = support(crop(ref, uem)), support(crop(hyp, uem))
    ref_gaps, hyp_gaps = gaps(ref, uem), gaps(hyp, uem)
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


def detection_error_rate(components: np.ndarray) -> float:
    fa, miss, total = np.asarray(components, dtype=np.float64)
    if total == 0:
        return 0.0 if fa + miss == 0 else 1.0
    return float((fa + miss) / total)
