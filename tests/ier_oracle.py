"""Identification error rate components, restated in numpy from the definition in DESIGN.md "Identification error" (test
infrastructure: the device scorer, ``der_score<*, true>`` in csrc/der.cu, is compared against it bit for bit).

pyannote.metrics' ``IdentificationErrorRate`` counts the same five components as ``DiarizationErrorRate`` over the same
elementary intervals, with one difference: a reference label and a hypothesis label are matched when their names are equal,
instead of by the mapping of maximal total co-occurrence.  So ``ier_components`` is ``oracle.der.der_components`` with the
``linear_sum_assignment`` step replaced by name equality, and ``protocol_ier_components`` is
``scoring_protocol.der_components`` with this scorer on the cropped annotations.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from diart_b200.core import Annotation, Segment
from oracle.der import activity
from scoring_protocol import crop_annotation, scored


def named_unions(annotation: Annotation) -> Tuple[list, List[List[Tuple[float, float]]]]:
    """(label names in string order, per label its non-empty segments sorted, touching or overlapping ones merged)"""
    by_label = {}
    for segment, _, label in annotation.itertracks(yield_label=True):
        if segment:
            by_label.setdefault(label, []).append((segment.start, segment.end))
    names = sorted(by_label, key=str)
    unions = []
    for label in names:
        merged = []
        for a, b in sorted(by_label[label]):
            if merged and a <= merged[-1][1]:
                merged[-1] = (merged[-1][0], max(merged[-1][1], b))
            else:
                merged.append((a, b))
        unions.append(merged)
    return names, unions


def ier_components(reference: Annotation, hypothesis: Annotation) -> np.ndarray:
    """float64 (5,) = false alarm, missed detection, confusion, correct, total (seconds), labels matched by name"""
    ref_names, ref = named_unions(reference)
    hyp_names, hyp = named_unions(hypothesis)
    bounds = np.unique(np.array([t for u in ref + hyp for seg in u for t in seg], dtype=np.float64))
    lo, hi = bounds[:-1], bounds[1:]
    keep = np.array([bool(Segment(a, b)) for a, b in zip(lo.tolist(), hi.tolist())], dtype=bool)
    lo, hi = lo[keep], hi[keep]
    d = hi - lo
    ar, ah = activity(ref, lo, hi), activity(hyp, lo, hi)
    nr, nh = ar.sum(axis=0), ah.sum(axis=0)
    c = np.zeros(len(d), dtype=np.int64)
    for r, name in enumerate(ref_names):
        if name in hyp_names:
            c += ar[r] & ah[hyp_names.index(name)]

    def seq(x):
        return float(np.cumsum(d * x)[-1]) if len(d) else 0.0

    return np.array([seq(np.maximum(0, nh - nr)), seq(np.maximum(0, nr - nh)), seq(np.minimum(nr, nh) - c), seq(c),
                     seq(nr)], dtype=np.float64)


def protocol_ier_components(reference: Annotation, hypothesis: Annotation, collar: float = 0.0, skip_overlap: bool = False,
                            uem: Optional[Sequence] = None) -> np.ndarray:
    """float64 (5,) of ``IdentificationErrorRate(collar, skip_overlap)(reference, hypothesis, uem=uem)``'s components: both
    sides cropped to the scored regions of DESIGN.md "DER scoring" steps 1-4, then :func:`ier_components`"""
    regions = scored(reference, hypothesis, collar, skip_overlap, uem)
    return ier_components(crop_annotation(reference, regions), crop_annotation(hypothesis, regions))
