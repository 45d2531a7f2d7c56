"""Known speakers: the speakers a pipeline or a live stream starts with.

:class:`KnownSpeakers` holds names and float64 centroids.  Given to ``SpeakerDiarization.set_known_speakers`` or
``MultiStreamDiarization.open(speakers=...)``, it becomes the clustering's initial state: centres 0 .. n - 1 hold the
centroids and are active, and the state counts as initialised.  The reference's ``OnlineSpeakerClustering.identify``
(``src/diart/blocks/clustering.py:149``) takes its first-chunk path only while ``centers is None``, so a pre-filled state goes
straight to the distance path: new local speakers are matched against the known centroids, those are updated with
``rho_update`` and new speakers are added after them.  Centre g < n is labelled ``names[g]``, every other centre
``speaker<g>``.

:func:`enroll` computes centroids from audio: one clip per name, the centroid the clustering holds for the clip's dominant
speaker at the end of the clip.  ``speakers()`` of a pipeline or a stream exports its state as a :class:`KnownSpeakers`, so a
stream can be closed and later resumed with the same centroids, bit for bit, and the same labels.

:class:`SpeakerGallery` names discovered speakers from an enrolled gallery of any size (DESIGN.md "Gallery naming"): a global
speaker that is not named yet takes the name of its nearest gallery entry by cosine distance, in float64, when that distance
is below the gallery's threshold and no other speaker of the same stream has that entry.
"""
from __future__ import annotations

import ctypes as C
import math
import re
import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .core import Annotation

_SPEAKER_LABEL = re.compile(r"speaker(0|[1-9][0-9]*)")


def check_names(names: Sequence[str]):
    """ValueError naming the first offending entry unless every name is a non-empty str without whitespace (names become
    RTTM fields), the names are unique, and a name ``speaker<j>`` sits at index j (so that it cannot be the label of a
    speaker the clustering discovers)"""
    seen = set()
    for i, name in enumerate(names):
        if not isinstance(name, str) or not name:
            raise ValueError(f"speaker {i}: the name must be a non-empty string, not {name!r}")
        if any(ch.isspace() for ch in name):
            raise ValueError(f"speaker {i}: the name {name!r} contains whitespace")
        if name in seen:
            raise ValueError(f"speaker {i}: the name {name!r} is given twice")
        m = _SPEAKER_LABEL.fullmatch(name)
        if m and int(m.group(1)) != i:
            raise ValueError(f"speaker {i}: the name {name!r} may only be given to speaker {m.group(1)}, whose default "
                             "label it is")
        seen.add(name)


class KnownSpeakers:
    """Names (tuple of str) and centroids (float64 (n, D), C-contiguous, read-only, owned), checked on construction:
    :func:`check_names`, one centroid per name, every centroid finite with a non-zero norm (a zero centroid has no cosine
    distance).  n = 0 means no known speakers.  Immutable."""

    __slots__ = ("names", "centroids")

    def __init__(self, names: Sequence[str], centroids):
        names = tuple(names)
        c = np.array(centroids, dtype=np.float64, order="C", copy=True)
        if c.size == 0 and c.ndim < 2:
            c = c.reshape(0, 0)
        if c.ndim != 2:
            raise ValueError(f"centroids must have shape (n, D), not {c.shape}")
        if len(names) != c.shape[0]:
            raise ValueError(f"{len(names)} names and {c.shape[0]} centroids")
        check_names(names)
        for i in range(c.shape[0]):
            if not np.all(np.isfinite(c[i])):
                raise ValueError(f"speaker {i} ({names[i]}): the centroid is not finite")
            if not np.dot(c[i], c[i]) > 0:
                raise ValueError(f"speaker {i} ({names[i]}): the centroid has a zero norm")
        c.setflags(write=False)
        object.__setattr__(self, "names", names)
        object.__setattr__(self, "centroids", c)

    def __setattr__(self, name, value):
        raise AttributeError("KnownSpeakers is immutable")

    def __len__(self) -> int:
        return len(self.names)

    @property
    def dimension(self) -> int:
        return int(self.centroids.shape[1])

    def __eq__(self, other) -> bool:
        return (isinstance(other, KnownSpeakers) and self.names == other.names
                and self.centroids.shape == other.centroids.shape
                and np.array_equal(self.centroids.view(np.int64), other.centroids.view(np.int64)))

    __hash__ = None

    def __repr__(self) -> str:
        return f"KnownSpeakers(names={list(self.names)}, dimension={self.dimension})"


def speaker_labels(known: Optional[KnownSpeakers], max_speakers: int) -> List[str]:
    """the label of every global speaker: ``names[g]`` for a known one, ``speaker<g>`` for the others"""
    names = known.names if known is not None else ()
    return [names[g] if g < len(names) else f"speaker{g}" for g in range(int(max_speakers))]


def exported(labels: Sequence[str], centers: np.ndarray, active: np.ndarray) -> KnownSpeakers:
    """a clustering state (centroids (M, D), active flags (M,)) -> its active centres with their labels.  The reference
    never deactivates a centre and always takes the lowest free one, so the active centres are a prefix 0 .. k - 1."""
    active = np.asarray(active) != 0
    k = int(active.sum())
    assert active[:k].all(), f"the active centres {np.flatnonzero(active).tolist()} are not a prefix"
    return KnownSpeakers(list(labels[:k]), centers[:k])


def dominant_speaker(annotation: Annotation, labels: Sequence[str]) -> Optional[int]:
    """the index in ``labels`` of the speaker with the greatest total duration in ``annotation`` (ties: the lowest index),
    or None when it has no speech"""
    index = {label: g for g, label in enumerate(labels)}
    total = np.zeros(len(labels))
    for segment, _, label in annotation.itertracks(yield_label=True):
        total[index[label]] += segment.duration
    if not np.any(total > 0):
        return None
    return int(np.argmax(total))


def enroll(config, clips: Sequence[Tuple[str, np.ndarray]], timing: Optional[Dict[str, float]] = None) -> KnownSpeakers:
    """One clip per speaker -> their :class:`KnownSpeakers`.  ``clips``: (name, 1-D float32 waveform at
    ``config.sample_rate``).

    All clips go through the networks in one pass (``tune.DatasetSweep``) and are clustered in one launch at the config's
    own thresholds (``DatasetSweep.sweep(keep_state=True)``).  A clip's dominant speaker is the global speaker with the
    greatest total duration in its prediction -- the Annotation ``DatasetSweep.run([{}])`` returns for it, which is what
    ``Benchmark.run_single`` gives for the clip at this config -- ties going to the lowest index.  Its centroid is that
    speaker's row of the clip's final clustering state; the rows are gathered on the device and only they are downloaded.
    ValueError naming the clip when a clip's prediction has no speech.  ``timing`` (optional): receives the seconds of the
    sweep's construction (network pass) and of the clustering and gather."""
    from .tune import DatasetSweep, trial_params

    clips = list(clips)
    names = [name for name, _ in clips]
    check_names(names)
    if not clips:
        return KnownSpeakers([], np.zeros((0, 0)))
    t0 = time.perf_counter()
    ds = DatasetSweep(config, [(name, wav, None) for name, wav in clips])
    t1 = time.perf_counter()
    params = trial_params([{}], config)
    out = ds.sweep(params, keep_state=True)
    labels = speaker_labels(None, config.max_speakers)
    predictions = ds._run(params, lambda _: out, ds.labels)     # the Annotations DatasetSweep.run([{}]) builds
    dominant = []
    for name, (prediction,) in zip(names, predictions):
        g = dominant_speaker(prediction, labels)
        if g is None:
            raise ValueError(f"clip {name!r}: its prediction has no speech, so it has no dominant speaker")
        dominant.append(g)
    files = torch.arange(len(clips), device=out.centers.device)
    rows = out.centers[files, 0, torch.tensor(dominant, device=out.centers.device)].cpu().numpy()
    if timing is not None:
        timing.update(construct=t1 - t0, sweep=time.perf_counter() - t1)
    return KnownSpeakers(names, rows)


def is_default_label(label: str, g: int) -> bool:
    """whether ``label`` is ``speaker<g>``, the label of a global speaker g that has no name"""
    return label == f"speaker{g}"


class SpeakerGallery:
    """Enrolled speakers to name discovered speakers from: ``known`` (a :class:`KnownSpeakers`, any number of entries up to
    2^20) and a cosine-distance ``threshold`` (0 < threshold <= 2), held on ``device`` as float64 (uploaded at first use).

    The naming rule, per stream (or per :meth:`name` call): every global speaker not named yet is compared with every entry
    the stream has not claimed; its nearest entry (ties: the lowest index) is a candidate when the distance is
    ``< threshold``.  Among candidates for one entry the smallest distance wins (ties: the lowest speaker index); the winner
    takes the entry's name for good and the entry is claimed; the others are compared again next time.  A speaker whose
    label is already a name (a known speaker) counts as named, and a gallery entry of that name as claimed.

    ValueError for a gallery name of the form ``speaker<j>`` (the label of a discovered speaker) or a bad threshold; the
    names and centroids are checked as :class:`KnownSpeakers` checks them."""

    def __init__(self, known: KnownSpeakers, threshold: float, device=None):
        if not isinstance(known, KnownSpeakers):
            raise TypeError(f"known: expected KnownSpeakers, got {type(known).__name__}")
        if not 1 <= len(known) <= 1 << 20:
            raise ValueError(f"a gallery holds 1 .. 1048576 entries, not {len(known)}")
        for e, name in enumerate(known.names):
            if _SPEAKER_LABEL.fullmatch(name):
                raise ValueError(f"entry {e}: the name {name!r} is the label of a discovered speaker")
        threshold = float(threshold)
        if not (math.isfinite(threshold) and 0 < threshold <= 2):
            raise ValueError(f"threshold must be finite and in (0, 2], not {threshold}")
        self.known, self.threshold = known, threshold
        self.device = torch.device("cuda") if device is None else torch.device(device)
        self.index = {name: e for e, name in enumerate(known.names)}
        self._h: Optional[C.c_void_p] = None

    def __len__(self) -> int:
        return len(self.known)

    @property
    def names(self) -> Tuple[str, ...]:
        return self.known.names

    @property
    def dimension(self) -> int:
        return self.known.dimension

    @property
    def handle(self) -> C.c_void_p:
        """the ``dg_gallery`` handle, created on first use"""
        if self._h is None:
            _lib.require_cuda(self.device)
            index = self.device.index if self.device.index is not None else torch.cuda.current_device()
            h = C.c_void_p()
            c = self.known.centroids
            _lib.check(_lib.lib().dg_gallery_create(c.ctypes.data, len(self), self.dimension, index, C.byref(h)))
            self._h = h
        return self._h

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                _lib.lib().dg_gallery_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    def claims(self, labels: Sequence[str]) -> Tuple[int, np.ndarray]:
        """the named speakers of a label list (bit g: ``labels[g]`` is not ``speaker<g>``) and the entry each one claims,
        int32 (len(labels),), -1 where the name is not in the gallery or the speaker is not named"""
        named, claimed = 0, np.full(len(labels), -1, dtype=np.int32)
        for g, label in enumerate(labels):
            if not is_default_label(label, g):
                named |= 1 << g
                claimed[g] = self.index.get(label, -1)
        return named, claimed

    def _query(self, x: np.ndarray, group: np.ndarray, claimed: Optional[np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
        dev = self.device
        x_d = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).to(dev)
        g_d = torch.from_numpy(np.ascontiguousarray(group, dtype=np.int32)).to(dev)
        c_d = None if claimed is None else torch.from_numpy(np.ascontiguousarray(claimed, dtype=np.int32)).to(dev)
        entry = torch.empty(len(x), dtype=torch.int32, device=dev)
        dist = torch.empty(len(x), dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().dg_gallery_query(self.handle, x_d.data_ptr(), len(x), g_d.data_ptr(), _lib.ptr(c_d),
                                                   self.threshold, entry.data_ptr(), dist.data_ptr(), _lib.stream_ptr(dev)))
        return entry.cpu().numpy().astype(np.int64), dist.cpu().numpy()

    def identify(self, centroids, claimed=None) -> Tuple[np.ndarray, np.ndarray]:
        """centroids float64 (Q, D) -> (entry int64 (Q,), distance float64 (Q,)): each row's nearest entry outside
        ``claimed`` (at most 32 entry indices; ties: the lowest index) and its distance, entry -1 where that distance is not
        below the threshold (distance +inf when every entry is claimed).  Rows are independent of each other."""
        x = np.asarray(centroids, dtype=np.float64)
        if x.ndim != 2 or x.shape[1] != self.dimension:
            raise ValueError(f"centroids must have shape (Q, {self.dimension}), not {x.shape}")
        row = np.full(32, -1, dtype=np.int32)
        if claimed is not None:
            c = np.asarray(claimed, dtype=np.int64).reshape(-1)
            if len(c) > 32 or np.any((c < 0) | (c >= len(self))):
                raise ValueError(f"claimed: at most 32 entry indices in [0, {len(self)})")
            row[:len(c)] = c
        if len(x) == 0:
            return np.zeros(0, dtype=np.int64), np.zeros(0)
        return self._query(x, np.arange(len(x)), np.tile(row, (len(x), 1)))

    def name(self, state: KnownSpeakers) -> KnownSpeakers:
        """``state`` (a pipeline's or a stream's ``speakers()``) with its ``speaker<g>`` entries named by the rule, as one
        tick of a stream names them"""
        if not isinstance(state, KnownSpeakers):
            raise TypeError(f"state: expected KnownSpeakers, got {type(state).__name__}")
        if len(state) == 0:
            return state
        if state.dimension != self.dimension:
            raise ValueError(f"the state's centroids have dimension {state.dimension}, the gallery {self.dimension}")
        if len(state) > 32:
            raise ValueError(f"{len(state)} speakers, at most 32")
        labels = list(state.names)
        named, claimed = self.claims(labels)
        rows = [g for g in range(len(labels)) if not (named >> g) & 1]
        if not rows:
            return state
        table = np.full((1, 32), -1, dtype=np.int32)
        taken = claimed[claimed >= 0]
        table[0, :len(taken)] = taken
        entry, _ = self._query(state.centroids[rows], np.zeros(len(rows)), table)
        for g, e in zip(rows, entry.tolist()):
            if e >= 0:
                labels[g] = self.names[e]
        return KnownSpeakers(labels, state.centroids)


def check_gallery(gallery: SpeakerGallery, config, dimension: int):
    """ValueError unless ``gallery`` can name the speakers of a server with ``config`` and embeddings of ``dimension``:
    the configuration compares speakers by cosine distance (centroids are unnormalised sums of embeddings, so only a
    scale-invariant distance compares a live centroid with an enrolled one), and the dimensions agree"""
    if not isinstance(gallery, SpeakerGallery):
        raise TypeError(f"gallery: expected SpeakerGallery or None, got {type(gallery).__name__}")
    metric = getattr(config, "metric", "cosine")
    if metric != "cosine":
        raise ValueError(f"a gallery names speakers by cosine distance; the configuration's metric is {metric!r}")
    if gallery.dimension != dimension:
        raise ValueError(f"the gallery's centroids have dimension {gallery.dimension}, the embeddings {dimension}")
