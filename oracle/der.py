"""Diarization error rate components, restated in numpy / scipy from the definition in DESIGN.md "DER scoring" (test
infrastructure: the device scorer, csrc/der.cu, is compared against it bit for bit).

Both sides: labels in string order, empty segments dropped, each label reduced to the union of its segments.  Elementary
intervals between consecutive distinct boundaries of both sides, skipped where ``Segment(b_i, b_i+1)`` is falsy; the label
mapping maximises the total co-occurrence (``scipy.optimize.linear_sum_assignment`` on its negation); every sum runs over the
intervals in time order, one float64 product added after another.
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np
from scipy.optimize import linear_sum_assignment

from diart_b200.core import Annotation, Segment

FIELDS = ("false_alarm", "missed_detection", "confusion", "correct", "total")


def label_unions(annotation: Annotation) -> List[List[Tuple[float, float]]]:
    """per label (string order) its non-empty segments, sorted, touching or overlapping ones merged"""
    by_label = {}
    for segment, _, label in annotation.itertracks(yield_label=True):
        if segment:
            by_label.setdefault(label, []).append((segment.start, segment.end))
    out = []
    for label in sorted(by_label, key=str):
        merged = []
        for a, b in sorted(by_label[label]):
            if merged and a <= merged[-1][1]:
                merged[-1] = (merged[-1][0], max(merged[-1][1], b))
            else:
                merged.append((a, b))
        out.append(merged)
    return out


def activity(unions: List[List[Tuple[float, float]]], lo: np.ndarray, hi: np.ndarray) -> np.ndarray:
    """bool (labels, intervals): label active over [lo, hi)"""
    act = np.zeros((len(unions), len(lo)), dtype=bool)
    for k, segs in enumerate(unions):
        for a, b in segs:
            act[k] |= (lo >= a) & (hi <= b)
    return act


def der_components(reference: Annotation, hypothesis: Annotation) -> np.ndarray:
    """float64 (5,) = false alarm, missed detection, confusion, correct, total (seconds)"""
    ref, hyp = label_unions(reference), label_unions(hypothesis)
    bounds = np.unique(np.array([t for u in ref + hyp for seg in u for t in seg], dtype=np.float64))
    lo, hi = bounds[:-1], bounds[1:]
    keep = np.array([bool(Segment(a, b)) for a, b in zip(lo.tolist(), hi.tolist())], dtype=bool)
    lo, hi = lo[keep], hi[keep]
    d = hi - lo
    ar, ah = activity(ref, lo, hi), activity(hyp, lo, hi)
    nr, nh = ar.sum(axis=0), ah.sum(axis=0)
    R, H = len(ref), len(hyp)
    c = np.zeros(len(d), dtype=np.int64)
    if R and H and len(d):
        # co-occurrence, each entry summed over the intervals in time order (cumsum accumulates sequentially)
        both = ar[:, None, :] & ah[None, :, :]
        C = np.cumsum(np.where(both, d[None, None, :], 0.0), axis=2)[:, :, -1]
        rows, cols = linear_sum_assignment(-C)
        for r, h in zip(rows, cols):
            c += ar[r] & ah[h]

    def seq(x):
        return float(np.cumsum(d * x)[-1]) if len(d) else 0.0

    return np.array([seq(np.maximum(0, nh - nr)), seq(np.maximum(0, nr - nh)), seq(np.minimum(nr, nh) - c), seq(c),
                     seq(nr)], dtype=np.float64)


def der(components: np.ndarray) -> float:
    fa, miss, conf, _, total = np.asarray(components, dtype=np.float64)
    num = fa + miss + conf
    if total == 0:
        return 0.0 if num == 0 else 1.0
    return float(num / total)
