"""Gallery naming restated in plain numpy float64 (DESIGN.md "Gallery naming"), for the host and GPU tests.

A stream's global speaker g is named when its label is not ``speaker<g>``.  After a tick, every active, unnamed speaker is
compared with every gallery entry the stream has not claimed (the entries named like one of its speakers); its nearest
entry by cosine distance 1 - clip(u.v / (|u| |v|), -1, 1), ties to the lowest index, is a candidate when the distance is
< threshold; among the candidates for one entry the smallest distance wins, ties to the lowest g.  Winners take the entry's
name; the others stay unnamed until the stream's next tick."""
import numpy as np


def first_copies(entries: np.ndarray) -> np.ndarray:
    """for each gallery row, the lowest index of a row bitwise equal to it"""
    _, first, inverse = np.unique(np.ascontiguousarray(entries).view(np.int64), axis=0, return_index=True,
                                  return_inverse=True)
    return first[inverse.reshape(-1)]


def cosine_distances(x: np.ndarray, entries: np.ndarray, copies=None) -> np.ndarray:
    """(Q, D), (G, D) -> (Q, G) float64; identical entries get identical columns (``copies``: ``first_copies(entries)``)"""
    x, entries = np.asarray(x, dtype=np.float64), np.asarray(entries, dtype=np.float64)
    c = (x @ entries.T) / (np.linalg.norm(x, axis=1)[:, None] * np.linalg.norm(entries, axis=1)[None, :])
    d = 1.0 - np.clip(c, -1.0, 1.0)
    copies = first_copies(entries) if copies is None else copies
    return d[:, copies]


def nearest(d: np.ndarray, claimed=()) -> tuple:
    """distances (Q, G), claimed entries -> (entry (Q,), distance (Q,), runner-up distance over the other distinct rows
    (Q,)); entry -1 / distance inf where every entry is claimed"""
    d = np.array(d, dtype=np.float64)
    d[:, list(claimed)] = np.inf
    entry = np.argmin(d, axis=1) if d.shape[1] else np.zeros(len(d), dtype=np.int64)
    best = d[np.arange(len(d)), entry] if d.shape[1] else np.full(len(d), np.inf)
    other = np.where(d == best[:, None], np.inf, d)
    runner = other.min(axis=1) if d.shape[1] else np.full(len(d), np.inf)
    entry = np.where(np.isfinite(best), entry, -1)
    return entry, best, runner


def resolve(entry: np.ndarray, dist: np.ndarray, threshold: float) -> np.ndarray:
    """the winners of one claim group: entry (Q,) where query q (in speaker order) wins it, else -1"""
    out = np.full(len(entry), -1, dtype=np.int64)
    for q in range(len(entry)):
        e = entry[q]
        if e < 0 or not dist[q] < threshold:
            continue
        rivals = [k for k in range(len(entry)) if k != q and entry[k] == e and dist[k] < threshold]
        if all((dist[q], q) < (dist[k], k) for k in rivals):
            out[q] = e
    return out


def is_named(label: str, g: int) -> bool:
    return label != f"speaker{g}"


def name_step(labels, centroids, names, entries, threshold, copies=None):
    """one tick of one stream: labels of its active speakers 0 .. k - 1 with centroids (k, D) -> (new labels, [(g, best
    distance, runner-up, threshold margin)] of the speakers compared)"""
    labels = list(labels)
    index = {name: e for e, name in enumerate(names)}
    claimed = [index[label] for g, label in enumerate(labels) if is_named(label, g) and label in index]
    rows = [g for g, label in enumerate(labels) if not is_named(label, g)]
    if not rows:
        return labels, []
    d = cosine_distances(np.asarray(centroids)[rows], entries, copies)
    entry, best, runner = nearest(d, claimed)
    won = resolve(entry, best, threshold)
    for g, e in zip(rows, won.tolist()):
        if e >= 0:
            labels[g] = names[e]
    return labels, [(g, best[i], runner[i], abs(best[i] - threshold)) for i, g in enumerate(rows)]
