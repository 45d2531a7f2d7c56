"""DER components on the host: oracle/der.py on hand-built cases with exact (dyadic) sums, its mapping against a brute force
over every one-to-one mapping, diart_b200.tune.reference_arrays and DERComponents."""
import itertools

import numpy as np
import pytest

from diart_b200.core import Annotation, Segment
from diart_b200.tune import DERComponents, reference_arrays
from oracle.der import activity, der, der_components, label_unions


def ann(spec):
    """{label: [(start, end), ...]} -> Annotation"""
    a = Annotation(uri="f")
    n = 0
    for label, segs in spec.items():
        for s, e in segs:
            a[Segment(s, e), n] = label
            n += 1
    return a


def comps(fa=0.0, miss=0.0, conf=0.0, corr=0.0, total=0.0):
    return np.array([fa, miss, conf, corr, total])


CASES = {
    "perfect under relabelling": ({"A": [(0, 2)], "B": [(1, 3)]}, {"x": [(0, 2)], "y": [(1, 3)]}, comps(corr=4, total=4), 0.0),
    "empty hypothesis": ({"A": [(0, 1.5)], "B": [(0.5, 2)]}, {}, comps(miss=3, total=3), 1.0),
    "false alarm only": ({"A": [(0, 1)]}, {"x": [(0, 1)], "y": [(2, 2.5)]}, comps(fa=0.5, corr=1, total=1), 0.5),
    "empty reference": ({}, {"x": [(0, 1)]}, comps(fa=1), 1.0),
    "both empty": ({}, {}, comps(), 0.0),
    "overlap with confusion": ({"A": [(0, 2)], "B": [(1, 3)]}, {"x": [(0, 1)], "y": [(1, 3)], "z": [(1, 1.5)]},
                               comps(miss=0.5, conf=0.5, corr=3, total=4), 0.25),
    "more hypothesis labels": ({"A": [(0, 4)]}, {"x": [(0, 1)], "y": [(1, 4)]}, comps(conf=1, corr=3, total=4), 0.25),
    "fewer hypothesis labels": ({"A": [(0, 1)], "B": [(1, 4)]}, {"x": [(0, 4)]}, comps(conf=1, corr=3, total=4), 0.25),
    "self-overlapping label is its union": ({"A": [(0, 2), (1, 3), (3, 3.5)]}, {"x": [(0, 3.5)]},
                                            comps(corr=3.5, total=3.5), 0.0),
}


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_hand_built_cases(name):
    ref, hyp, want, want_der = CASES[name]
    got = der_components(ann(ref), ann(hyp))
    assert np.array_equal(got, want), (got, want)
    assert der(got) == want_der
    assert DERComponents.from_array(got[None]).der[0] == want_der


def brute_force_der(ref: Annotation, hyp: Annotation) -> float:
    """the smallest DER over every one-to-one mapping of the labels, with the oracle's intervals"""
    ru, hu = label_unions(ref), label_unions(hyp)
    bounds = np.unique([t for u in ru + hu for seg in u for t in seg])
    lo, hi = bounds[:-1], bounds[1:]
    d = hi - lo
    ar, ah = activity(ru, lo, hi), activity(hu, lo, hi)
    nr, nh = ar.sum(0), ah.sum(0)
    base = float(np.sum(d * np.maximum(0, nh - nr)) + np.sum(d * np.maximum(0, nr - nh)) + np.sum(d * np.minimum(nr, nh)))
    total = float(np.sum(d * nr))
    best = np.inf
    R, H = len(ru), len(hu)
    pairs = ([list(zip(range(R), p)) for p in itertools.permutations(range(H), R)] if R <= H else
             [list(zip(p, range(H))) for p in itertools.permutations(range(R), H)])
    for mapping in pairs or [[]]:
        c = np.zeros(len(d), dtype=np.int64)
        for r, h in mapping:
            c += ar[r] & ah[h]
        num = base - float(np.sum(d * c))
        best = min(best, (0.0 if num == 0 else 1.0) if total == 0 else num / total)
    return best


def random_annotation(rng, n_labels, names):
    spec = {}
    for k in range(n_labels):
        n = rng.integers(1, 5)
        t = np.sort(rng.integers(0, 64, 2 * n)) / 4.0        # quarter seconds: every sum is exact
        spec[names[k]] = [(a, b) for a, b in zip(t[0::2], t[1::2]) if b > a]
    return ann(spec)


@pytest.mark.parametrize("seed", range(40))
def test_oracle_mapping_is_optimal_by_brute_force(seed):
    rng = np.random.default_rng(seed)
    ref = random_annotation(rng, int(rng.integers(0, 6)), [f"spk{i}" for i in range(5)])
    hyp = random_annotation(rng, int(rng.integers(0, 6)), [f"speaker{i}" for i in range(5)])
    got = der_components(ref, hyp)
    fa, miss, conf, corr, total = got
    assert miss + conf + corr == total                  # every reference second is counted once
    assert der(got) == brute_force_der(ref, hyp)


def test_reference_arrays():
    a = Annotation(uri="f")
    a[Segment(5, 6), 0] = "b"
    a[Segment(1, 3), 1] = "b"
    a[Segment(2, 4), 2] = "b"                     # overlaps the previous one: union
    a[Segment(4, 4.5), 3] = "b"                   # touches it: union
    a[Segment(0, 1), 4] = "a"
    a[Segment(7, 7 + 1e-7), 5] = "a"              # empty (Segment.__bool__): dropped
    a[Segment(3, 3.5), 6] = 10
    a[Segment(0.5, 1.5), 7] = "9"
    rows, labels, names = reference_arrays(a)
    assert names == [10, "9", "a", "b"]          # string order
    assert labels.dtype == np.int32 and rows.dtype == np.float64
    assert labels.tolist() == [0, 1, 2, 3, 3]
    assert rows.tolist() == [[3, 3.5], [0.5, 1.5], [0, 1], [1, 4.5], [5, 6]]


def test_reference_arrays_rejects_33_labels():
    ok = ann({f"s{i}": [(i, i + 1)] for i in range(32)})
    assert len(reference_arrays(ok)[2]) == 32
    with pytest.raises(ValueError, match="33 labels"):
        reference_arrays(ann({f"s{i}": [(i, i + 1)] for i in range(33)}))


def test_components_sum_and_der_rule():
    a = DERComponents.from_array(np.array([[1.0, 0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0, 0.0], [0.5, 0.25, 0.25, 3.0, 4.0]]))
    assert a.der.tolist() == [1.0, 0.0, 0.25]
    b = DERComponents.from_array(np.array([[0.0, 1.0, 0.0, 1.0, 2.0], [0.0, 0.0, 0.0, 2.0, 2.0], [0.0, 0.0, 0.0, 4.0, 4.0]]))
    s = a + b
    assert s.total.tolist() == [2.0, 2.0, 8.0]
    assert s.der.tolist() == [1.0, 0.0, 0.125]
    assert np.array_equal(s.as_array(), a.as_array() + b.as_array())
