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
"""
from __future__ import annotations

import re
import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

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
