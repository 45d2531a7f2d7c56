"""Hyper-parameter sweep of ``SpeakerDiarization`` on the device: one network pass per file, many trials per clustering launch.

The reference tunes ``tau_active``, ``rho_update`` and ``delta_new`` (``SpeakerDiarization.hyper_parameters()``) with
``diart.tune``: ``Optimizer.objective`` (reference ``src/diart/optim.py:98-122``) runs a full ``Benchmark`` per trial, i.e. the
segmentation and embedding networks once per trial and file.  None of the three parameters reaches the networks -- they
are read by the clustering (``blocks/clustering.py:137-142,168``) and by ``Binarize(tau_active)`` only.  So here a file
goes through the networks ONCE (the fused pipeline, batches of 256) and ``dg_sweep_run`` clusters and post-processes the
resulting scores and embeddings for T trials at once (one CTA per trial state, ``csrc/cluster.cu``; one CTA per chunk
and trial, ``csrc/post.cu``).

For each trial :meth:`HyperParameterSweep.run` returns what ``Benchmark.run_single`` (``inference.py:308-357``) returns
for a pipeline with that trial's parameters: the whole-file prediction that ``PredictionAccumulator(uri)`` (patch
collar 0.05 s) collects over the per-chunk outputs, assembled from the packed turn list without building per-chunk
annotations.

:meth:`HyperParameterSweep.score` goes one step further and returns what ``Benchmark.evaluate`` (``inference.py:359-390``)
computes from those predictions: the diarization error rate components of every trial against a reference
(``DiarizationErrorRate(collar=0, skip_overlap=False)``; definition in DESIGN.md "DER scoring"), evaluated on the device by
``dg_sweep_score`` (``csrc/der.cu``) without building any ``Annotation``.  :meth:`HyperParameterSweep.score_files` sums them over
files: its ``total.der`` is the value ``Optimizer.objective`` minimises.

:class:`DatasetSweep` does the same for a whole dataset at once: the network pass of every file runs once, in one pipelined
flow, and its outputs stay on the device; every ``score`` / ``run`` call then clusters, post-processes and scores all
(file, trial) pairs in one launch per kernel (``dg_sweep_score_files`` / ``dg_sweep_run_files``), without running a network
kernel again.

:class:`VoiceActivitySweep` does it for ``VoiceActivityDetection``, whose one hyper-parameter, ``tau_active``, is read by
``Binarize`` alone: the segmentation runs once per dataset, the aggregated speech curve is computed once per chunk
(``dg_vad_sweep_curve``, ``csrc/vad.cu``), and every trial only thresholds it and is scored by detection error rate
(``DetectionErrorRate(collar=0, skip_overlap=False)``, the pipeline's ``suggest_metric()``; DESIGN.md "Detection error").

Every ``score`` method also takes a ``metric`` (:class:`DiarizationErrorRate` / :class:`DetectionErrorRate`, or
pyannote.metrics' own, with a forgiveness collar and ``skip_overlap``) and the dataset sweeps a uem per file
(``uems``): :func:`scored_regions` computes each file's scored regions once, the references are cropped to them on the
host and the hypotheses on the device (``dg_sweep_set_scored_regions``; DESIGN.md "DER scoring", steps 1-5).

:class:`DatasetSweep` also tunes the overlap-aware embedding parameters ``gamma``, ``beta`` and
``normalize_embedding_weights`` (``osp=``): they reach the networks only at the embedding's statistics pooling, so one network
pass computes the scores once and the embeddings of every constructed *OSP set* (``dg_pipeline_nets_sets``), and each trial's
clustering reads the embeddings of its own set (``dg_sweep_set_trial_sets``; DESIGN.md "Sweeps over overlap-aware
weightings").

With known speakers (``DatasetSweep(..., speakers=...)``, :class:`~diart_b200.speakers.KnownSpeakers` per file) every
(file, trial) clustering starts from the file's centroids, as ``SpeakerDiarization.set_known_speakers`` starts a pipeline
(``dg_sweep_set_seeds``), and the speakers carry their names.  :class:`IdentificationErrorRate` then scores whether the names
are right: the DER components with each reference label matched to the hypothesis label of the same name instead of by the
optimal mapping (``dg_sweep_set_identities``; DESIGN.md "Identification error").

The three classes share their mechanics: :class:`FileBatches` cuts the window batches of every network pass,
:func:`stream_plan` is the post-path plan of one file, ``_timed`` puts CUDA events around one C call and ``_turn_list_call``
downloads a turn list into a host buffer that grows on demand.  ``HyperParameterSweep._run_trials`` / ``_score_trials`` are the
bodies of the one-file and the ``_files`` entry points of the diarization sweep, and ``_DatasetSweep`` is the base of the two
dataset classes (files, offsets, plans, references and the loops over trial groups).
"""
from __future__ import annotations

import bisect
import copy
import ctypes as C
import functools
import itertools
import math
import operator
import time
from dataclasses import dataclass
from typing import Dict, Iterable, List, Mapping, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .blocks.diarization import SpeakerDiarization, SpeakerDiarizationConfig
from .blocks.post import post_plan, turn_times
from .blocks.vad import VoiceActivityDetection, VoiceActivityDetectionConfig
from .core import Annotation, Segment
from .models import B200PyanNet
from .operators import DeviceAudioStream
from .speakers import KnownSpeakers, speaker_labels

NETWORK_BATCH = 256           # windows per network step (the benchmarked batch)
STREAM_FORM_MIN_BATCH = 4     # the sinc front end's stream form runs for batches of this many windows on (api_seg.cu)
TRIALS_PER_LAUNCH = 1024      # trials per dg_sweep_run; more run as further launches over the same network outputs
TRIAL_CHUNKS_PER_LAUNCH = 4 << 20   # DatasetSweep: trials x chunks per launch (bounds the header, maps and turn buffers)
PATCH_COLLAR = 0.05           # PredictionAccumulator's default (sinks.py)
MAX_REFERENCE_LABELS = 32     # one lane per reference label in the scoring kernel
PRECISION = 1e-6              # pyannote.core's SEGMENT_PRECISION: Segment.__bool__, Segment.intersects
MAX_OSP_SETS = 64            # OSP sets per network pass (dg_pipeline_nets_sets)
WHOLE_LINE = (-1e300, 1e300)  # the uem of a file that has none (scored_regions: the scored regions do not depend on the trial)


def trial_params(trials: Sequence[Mapping[str, float]], config, names: Optional[Sequence[str]] = None) -> np.ndarray:
    """trials (dicts keyed by the reference's HyperParameter names) -> float64 (T, len(names)), by default names =
    {tau_active, rho_update, delta_new} (``SpeakerDiarization.hyper_parameters()``); a missing key takes the config's value.
    Other keys (gamma, beta, latency, step, max_speakers, ...) change the network pass or the plan and cannot vary within
    one sweep: ValueError."""
    names = list(names) if names is not None else [hp.name for hp in SpeakerDiarization.hyper_parameters()]
    trials = list(trials)
    if not trials:
        raise ValueError("at least one trial is needed")
    out = np.empty((len(trials), len(names)), dtype=np.float64)
    for i, trial in enumerate(trials):
        unknown = sorted(set(trial) - set(names))
        if unknown:
            raise ValueError(f"trial {i}: {unknown} cannot be swept (only {names}; the others change the network pass or "
                             f"the plan and stay fixed per sweep)")
        out[i] = [float(trial.get(n, getattr(config, n))) for n in names]
    return out


OSP_PARAMS = ("gamma", "beta", "normalize_embedding_weights")   # the config keys of an OSP set


def osp_set(entry: Mapping, config) -> Tuple[float, float, bool]:
    """one OSP set -> (gamma, beta, normalize) as the pipeline receives them: gamma and beta rounded to float32, a missing key
    the config's value.  ValueError for another key or a non-finite gamma / beta."""
    unknown = sorted(set(entry) - set(OSP_PARAMS))
    if unknown:
        raise ValueError(f"OSP set {dict(entry)}: unknown keys {unknown} (only {list(OSP_PARAMS)})")
    values = [float(entry.get(n, getattr(config, n))) for n in OSP_PARAMS[:2]]
    if not all(math.isfinite(v) for v in values):
        raise ValueError(f"OSP set {dict(entry)}: gamma and beta must be finite")
    gamma, beta = (float(np.float32(v)) for v in values)
    return gamma, beta, bool(entry.get(OSP_PARAMS[2], config.normalize_embedding_weights))


def osp_sets(config, osp: Iterable[Mapping] = ()) -> Tuple[Tuple[float, float, bool], ...]:
    """the OSP sets a sweep constructs: the config's own first, then those of ``osp`` (entries keyed like the config, see
    :func:`osp_set`) in order, duplicates (equal float32 gamma and beta, equal normalize) once"""
    out = [osp_set({}, config)]
    for entry in osp:
        s = osp_set(entry, config)
        if s not in out:
            out.append(s)
    if len(out) > MAX_OSP_SETS:
        raise ValueError(f"{len(out)} OSP sets; at most {MAX_OSP_SETS} per sweep")
    return tuple(out)


def osp_index(config, sets: Sequence[Tuple[float, float, bool]], entry: Mapping) -> int:
    """the index in ``sets`` of the OSP set ``entry`` (:func:`osp_set`), else ValueError naming the constructed sets"""
    s = osp_set(entry, config)
    if s not in sets:
        raise ValueError(f"OSP set {osp_dict(s)} was not constructed (the sweep's sets: {[osp_dict(x) for x in sets]})")
    return list(sets).index(s)


def osp_dict(s: Tuple[float, float, bool]) -> Dict[str, object]:
    """(gamma, beta, normalize) -> the config-keyed dict of that set"""
    return dict(zip(OSP_PARAMS, s))


def trial_osp_params(trials: Sequence[Mapping[str, float]], config,
                     sets: Sequence[Tuple[float, float, bool]]) -> Tuple[np.ndarray, np.ndarray]:
    """trials that may also carry ``gamma``, ``beta`` and ``normalize_embedding_weights`` -> (each trial's OSP set index in
    ``sets`` int32 (T,), :func:`trial_params` of the rest float64 (T, 3)).  ValueError for a set that is not in ``sets``."""
    trials = list(trials)
    index = np.empty(len(trials), dtype=np.int32)
    rest = []
    for i, trial in enumerate(trials):
        try:
            index[i] = osp_index(config, sets, {k: trial[k] for k in OSP_PARAMS if k in trial})
        except ValueError as e:
            raise ValueError(f"trial {i}: {e}") from None
        rest.append({k: v for k, v in trial.items() if k not in OSP_PARAMS})
    return index, trial_params(rest, config)


def trial_osp_sets(config, trials: Sequence[Mapping[str, float]]) -> Tuple[Tuple[float, float, bool], ...]:
    """:func:`osp_sets` of the distinct OSP sets the trials name (the config's own first)"""
    return osp_sets(config, [{k: t[k] for k in OSP_PARAMS if k in t} for t in trials])


def _set_trial_sets(handle, trial_sets: Optional[Tuple[int, np.ndarray]]):
    """the handle's trial sets for its next call: (number of sets, int32 (T,) set per trial), or None (embeddings of one set)"""
    if trial_sets is None:
        _lib.check(_lib.lib().dg_sweep_set_trial_sets(handle, 0, None, 0))
    else:
        G, index = trial_sets
        index = np.ascontiguousarray(index, dtype=np.int32)
        _lib.check(_lib.lib().dg_sweep_set_trial_sets(handle, int(G), index.ctypes.data, len(index)))


def _set_seeds(handle, seeds: Optional[Tuple[np.ndarray, np.ndarray]]):
    """the handle's known centroids for its next clustering calls: (offsets int32 (files + 1,), centroids float64 (n, D)) per
    clustering file, or None (every state starts fresh)"""
    if seeds is None:
        _lib.check(_lib.lib().dg_sweep_set_seeds(handle, 0, None, None))
    else:
        offsets, centers = seeds
        _lib.check(_lib.lib().dg_sweep_set_seeds(handle, len(offsets) - 1, offsets.ctypes.data, centers.ctypes.data))


def _set_identities(handle, table: Optional[np.ndarray]):
    """the handle's name matching for its next scoring calls: :func:`pack_identities`' table, or None (DER)"""
    if table is None:
        _lib.check(_lib.lib().dg_sweep_set_identities(handle, 0, None))
    else:
        _lib.check(_lib.lib().dg_sweep_set_identities(handle, len(table), table.ctypes.data))


@dataclass
class FileWindows:
    """What ``FileAudioSource`` + ``rearrange_audio_stream`` make of one file."""
    samples: np.ndarray       # the padded file, zero-filled to whole blocks of `step` samples
    offset: int               # first sample of window 0
    num_windows: int
    starts: np.ndarray        # float64 (num_windows,) start time of each window (before the timestamp shift)
    padding: tuple            # (left, right) seconds, config.get_file_padding
    chunk_samples: int
    step_samples: int

    def window(self, i: int) -> np.ndarray:
        a = self.offset + i * self.step_samples
        return self.samples[a:a + self.chunk_samples]


def file_windows(waveform: np.ndarray, config: SpeakerDiarizationConfig) -> FileWindows:
    """The windows ``Benchmark.run_single`` feeds a pipeline for a 1-D waveform at ``config.sample_rate``: padding from
    ``config.get_file_padding`` (reference ``inference.py:332``), blocks of ``step`` seconds with the last incomplete one
    zero-padded (``sources.py:88-127``), then ``rearrange_audio_stream``'s windows (``operators.py:44-100``)."""
    x = np.asarray(waveform, dtype=np.float32)
    if x.ndim != 1:
        raise ValueError(f"expected a 1-D waveform, got shape {x.shape}")
    sr = config.sample_rate
    left, right = config.get_file_padding(file_duration=len(x) / sr)
    n_left = int(np.rint(left * sr)) if left > 0 else 0
    n_right = int(np.rint(right * sr)) if right > 0 else 0
    block = int(np.rint(config.step * sr))                    # FileAudioSource(block_duration=step)
    chunk, step = int(round(sr * config.duration)), int(round(sr * config.step))
    n = n_left + len(x) + n_right
    n_blocks = -(-n // block)
    samples = np.zeros(n_blocks * block, dtype=np.float32)
    samples[n_left:n_left + len(x)] = x
    # rearrange_audio_stream: each block of `step` samples extends the chunk; once it holds more than `chunk` samples it is
    # truncated to the last `chunk` and its start time advances by `step`; a chunk of exactly `chunk` samples is emitted
    first = -(-chunk // step)                                 # blocks until the first emission
    num_windows = max(0, n_blocks - first + 1)
    t, starts = 0.0, np.empty(num_windows)
    if first * step > chunk:
        t += config.step
    for i in range(num_windows):
        if i:
            t += config.step
        starts[i] = t
    return FileWindows(samples, first * step - chunk, num_windows, starts, (left, right), chunk, step)


def assemble_predictions(header: np.ndarray, turns: np.ndarray, n_turns: int, out_start: np.ndarray, out_res: np.ndarray,
                         labels: Sequence[str], shift: float = 0.0, uri: Optional[str] = None,
                         collar: float = PATCH_COLLAR) -> List[Annotation]:
    """header int32 (T, N, 4) + packed turns of T trials over the same N chunks -> per trial the whole-file prediction of
    ``PredictionAccumulator(uri, collar)`` over that trial's per-chunk annotations (``DevicePostPath.annotations``).

    Vectorised ``Annotation.support(collar)`` (``core.py``): per trial and label (labels in string order), segments sorted
    by (start, end); a segment joins the current one when it starts before its end or less than ``collar`` after it."""
    T, N = header.shape[:2]
    row, g, s, e = turn_times(header.reshape(T * N, 4), turns, n_turns, out_start, out_res, shift)
    live = (e - s) > 1e-6                                     # Annotation drops empty segments (Segment.__bool__)
    row, g, s, e = row[live], g[live], s[live], e[live]
    trial = row // N
    M = len(labels)
    rank = np.empty(M, dtype=np.int64)
    rank[sorted(range(M), key=lambda i: str(labels[i]))] = np.arange(M)
    order = np.lexsort((e, s, rank[g], trial))
    trial, g, s, e = trial[order], g[order], s[order], e[order]
    gid = trial * M + rank[g]
    # running maximum of the ends within each (trial, label) group: ranks of the end values, offset per group, so that one
    # integer maximum-scan restarts at every group
    u, inv = np.unique(e, return_inverse=True)
    span = np.int64(len(u))
    cm = u[np.maximum.accumulate(gid * span + inv) - gid * span]
    first = np.ones(len(s), dtype=bool)
    first[1:] = gid[1:] != gid[:-1]
    prev = np.empty_like(cm)
    prev[0:1] = 0.0
    prev[1:] = cm[:-1]
    joins = ~first & ((s - prev < collar) | (s <= prev))
    heads = np.flatnonzero(~joins)
    tails = np.append(heads[1:], len(s))[:len(heads)] - 1
    m_start, m_end, m_trial, m_g = s[heads].tolist(), cm[tails].tolist(), trial[heads].tolist(), g[heads].tolist()
    modality = "speech" if shift == 0 else None               # what the first per-chunk annotation carries
    out = [Annotation(uri=uri, modality=modality) for _ in range(T)]
    track = [0] * T
    for a, b, t, k in zip(m_start, m_end, m_trial, m_g):
        out[t][Segment(a, b), track[t]] = labels[k]
        track[t] += 1
    return out


# ---------------------------------------------------------------------- scoring protocols (DESIGN.md "DER scoring", steps 1-4)
@dataclass(frozen=True)
class DiarizationErrorRate:
    """The constructor arguments of pyannote.metrics' ``DiarizationErrorRate`` a diarization sweep can score with: a
    forgiveness ``collar`` (seconds, removed around every reference boundary, half on each side) and ``skip_overlap``
    (leave out the reference's overlapped speech).  The default is the pipelines' ``suggest_metric()``."""
    collar: float = 0.0
    skip_overlap: bool = False


@dataclass(frozen=True)
class IdentificationErrorRate:
    """The same for pyannote.metrics' ``IdentificationErrorRate``: DER's components with the labels matched by name instead
    of by the optimal mapping, for a :class:`DatasetSweep` whose speakers carry names (``speakers=``).  Only unit weights
    (pyannote's ``confusion``, ``miss`` and ``false_alarm`` arguments) are supported."""
    collar: float = 0.0
    skip_overlap: bool = False


@dataclass(frozen=True)
class DetectionErrorRate:
    """The same for pyannote.metrics' ``DetectionErrorRate``, the metric of :class:`VoiceActivitySweep`."""
    collar: float = 0.0
    skip_overlap: bool = False


def metric_protocol(metric, kind: str) -> Tuple[float, bool]:
    """``metric`` (None: the default) -> (collar, skip_overlap).  Accepted: an object whose class is named ``kind``
    (:class:`DiarizationErrorRate` / :class:`DetectionErrorRate`, or pyannote.metrics' class of that name) with ``collar``
    and ``skip_overlap`` attributes; the collar must be a finite number >= 0.  Anything else: ValueError."""
    if metric is None:
        return 0.0, False
    if type(metric).__name__ != kind or not hasattr(metric, "collar") or not hasattr(metric, "skip_overlap"):
        raise ValueError(f"metric {metric!r}: this sweep scores a {kind} (collar, skip_overlap)")
    collar = metric.collar
    if isinstance(collar, bool) or not isinstance(collar, (int, float, np.integer, np.floating)) or \
            not math.isfinite(float(collar)) or float(collar) < 0:
        raise ValueError(f"metric collar {collar!r}: need a finite number >= 0")
    return float(collar), bool(metric.skip_overlap)


IER_WEIGHTS = ("confusion", "miss", "false_alarm")   # pyannote's IdentificationErrorRate weights; only 1 is supported


def diarization_metric(metric) -> Tuple[str, float, bool]:
    """``metric`` of a :class:`DatasetSweep` (None: the default) -> (its class name, collar, skip_overlap): a
    :class:`DiarizationErrorRate` or an :class:`IdentificationErrorRate` (or pyannote.metrics' class of either name) as
    :func:`metric_protocol` accepts them; an identification error rate whose ``confusion``, ``miss`` or ``false_alarm``
    weight is not 1: ValueError."""
    kind = "IdentificationErrorRate" if type(metric).__name__ == "IdentificationErrorRate" else "DiarizationErrorRate"
    if kind == "IdentificationErrorRate":
        for name in IER_WEIGHTS:
            w = getattr(metric, name, 1.0)
            if isinstance(w, bool) or not isinstance(w, (int, float, np.integer, np.floating)) or float(w) != 1.0:
                raise ValueError(f"metric {name} weight {w!r}: only unit weights are supported")
    return (kind, *metric_protocol(metric, kind))


def check_uem(uem) -> Optional[List[Tuple[float, float]]]:
    """A uem (None, or a list of ``(start, end)`` pairs or ``Segment``s sorted by (start, end), each finite and truthy)
    -> a list of float pairs; anything else: ValueError"""
    if uem is None:
        return None
    if not isinstance(uem, (list, tuple)):
        raise ValueError(f"a uem is a list of (start, end) pairs or Segments, not {type(uem).__name__}")
    out = []
    for i, piece in enumerate(uem):
        try:
            start, end = (piece.start, piece.end) if hasattr(piece, "start") else piece
            start, end = float(start), float(end)
        except (TypeError, ValueError):
            raise ValueError(f"uem piece {i} ({piece!r}) is not a (start, end) pair or a Segment") from None
        if not (math.isfinite(start) and math.isfinite(end)) or not end - start > PRECISION:
            raise ValueError(f"uem piece {i} ({start}, {end}) is not finite or not longer than {PRECISION} s (falsy)")
        out.append((start, end))
    if out != sorted(out):
        raise ValueError("the uem pieces are not sorted by (start, end)")
    return out


def _truthy(a: float, b: float) -> bool:
    """``bool(Segment(a, b))``"""
    return (b - a) > PRECISION


def _co_iter(a: List[Tuple[float, float]], b: List[Tuple[float, float]]):
    """``Timeline.co_iter``: pairs (x, y), x of sorted ``a`` in order, y of sorted ``b`` in order, with ``x.intersects(y)``
    (pyannote.core's rule).  The y before the first whose running maximum of ends reaches x's start end before x starts,
    so cannot intersect it: they are skipped by bisection."""
    ends = list(itertools.accumulate((y[1] for y in b), max))
    for x in a:
        for y in b[bisect.bisect_left(ends, x[0]):]:
            if y > (x[1], x[1]):
                break
            if (x[0] < y[0] and y[0] < x[1] - PRECISION) or (x[0] > y[0] and x[0] < y[1] - PRECISION) or x[0] == y[0]:
                yield x, y


def _support(segs) -> List[Tuple[float, float]]:
    """``Timeline.support()`` of the unique segments in (start, end) order"""
    out: List[Tuple[float, float]] = []
    for s in sorted(set(segs)):
        if out and not _truthy(min(s[1], out[-1][1]), max(s[0], out[-1][0])):
            out[-1] = (min(out[-1][0], s[0]), max(out[-1][1], s[1]))
        else:
            out.append(s)
    return out


def _gaps(segs, uem) -> List[Tuple[float, float]]:
    """``Timeline(segs).gaps(support=uem)``: per piece of the uem's support, the truthy gaps between the support of the
    segments cropped to it"""
    out = []
    for u in _support(uem):
        end = u[0]
        inside = [(max(x[0], y[0]), min(x[1], y[1])) for x, y in _co_iter(sorted(set(segs)), [u])]
        for s in _support(p for p in inside if _truthy(*p)):
            if _truthy(end, s[0]):
                out.append((end, s[0]))
            end = s[1]
        if _truthy(end, u[1]):
            out.append((end, u[1]))
    return out


def scored_regions(reference: Annotation, collar: float = 0.0, skip_overlap: bool = False,
                   uem=None) -> List[Tuple[float, float]]:
    """The regions of a file that pyannote.metrics scores with ``collar`` / ``skip_overlap`` within ``uem`` (steps 1-3 of
    DESIGN.md "DER scoring"): the gaps, within the uem, of the support of the removed regions -- a ``collar``-wide segment
    around both ends of every unique non-empty reference segment, and the intersection of every pair of intersecting
    reference tracks other than a track with itself.  Sorted, each truthy, apart by more than 1e-6 s.

    Without a uem pyannote takes the extent of both sides, which depends on the hypothesis.  Nothing is active outside
    it, so the regions are computed within :data:`WHOLE_LINE` instead, once per file: the same scores except where a
    removed region starts within 1e-6 s of the extent's end or ends within 1e-6 s of its start (out of contract)."""
    collar, skip_overlap = metric_protocol(DiarizationErrorRate(collar, skip_overlap), "DiarizationErrorRate")
    uem = check_uem(uem)
    tracks: Dict[Tuple[float, float], int] = {}
    for segment, _ in reference.itertracks():
        if segment:
            key = (segment.start, segment.end)
            tracks[key] = tracks.get(key, 0) + 1
    segs = sorted(tracks)
    removed = []
    if collar > 0:
        for s, e in segs:
            removed += [(s - .5 * collar, s + .5 * collar), (e - .5 * collar, e + .5 * collar)]
    if skip_overlap:
        for x, y in _co_iter(segs, segs):
            if x != y or tracks[x] > 1:           # every pair of tracks but a track with itself
                removed.append((max(x[0], y[0]), min(x[1], y[1])))
    return _gaps(_support(r for r in removed if _truthy(*r)), [WHOLE_LINE] if uem is None else uem)


def cropped_tracks(annotation: Annotation, regions: Optional[Sequence[Tuple[float, float]]] = None) -> List[tuple]:
    """(start, end, label) of every non-empty track; with ``regions`` (sorted, apart) each cut against every region it
    intersects, the falsy pieces dropped: ``annotation.crop(regions, mode="intersection")`` (step 4)"""
    rows = [(s.start, s.end, label) for s, _, label in annotation.itertracks(yield_label=True) if s]
    if regions is None:
        return rows
    labels: Dict[Tuple[float, float], list] = {}
    for a, b, label in rows:
        labels.setdefault((a, b), []).append(label)
    out = []
    for x, r in _co_iter(sorted(labels), list(regions)):
        a, b = max(x[0], r[0]), min(x[1], r[1])
        if _truthy(a, b):
            out += [(a, b, label) for label in labels[x]]
    return out


def pack_regions(regions: Sequence[Sequence[Tuple[float, float]]]) -> Tuple[np.ndarray, np.ndarray]:
    """per-file scored regions -> the arguments of dg_sweep_set_scored_regions: (rows float64 (S, 2), offsets int32
    (files + 1,))"""
    rows = [np.asarray(r, dtype=np.float64).reshape(-1, 2) for r in regions]
    return (np.ascontiguousarray(np.concatenate(rows), dtype=np.float64),
            np.array(np.cumsum([0] + [len(r) for r in rows]), dtype=np.int32))


def reference_arrays(annotation: Annotation, regions: Optional[Sequence[Tuple[float, float]]] = None) \
        -> Tuple[np.ndarray, np.ndarray, List]:
    """A reference annotation -> (rows float64 (S, 2) start / end, labels int32 (S,), label names) for ``dg_sweep_score``:
    labels numbered in string order, empty segments dropped (``Segment.__bool__``), each label reduced to the union of its
    segments (rows of one label sorted, touching or overlapping segments merged).  With ``regions`` (:func:`scored_regions`)
    every segment is first cropped to them (:func:`cropped_tracks`); a label left without a piece disappears.

    pyannote.metrics scores a reference as given; where one label overlaps itself it may count that label twice in the
    overlap.  The union counts it once: the two agree for every reference in which no label overlaps itself.
    More than 32 labels: ValueError."""
    by_label: Dict = {}
    for start, end, label in cropped_tracks(annotation, regions):
        by_label.setdefault(label, []).append((start, end))
    names = sorted(by_label, key=str)
    if len(names) > MAX_REFERENCE_LABELS:
        raise ValueError(f"the reference has {len(names)} labels; at most {MAX_REFERENCE_LABELS} can be scored")
    rows, labels = [], []
    for r, name in enumerate(names):
        segs = sorted(by_label[name])
        cur_s, cur_e = segs[0]
        for a, b in segs[1:]:
            if a <= cur_e:
                cur_e = max(cur_e, b)
            else:
                rows.append((cur_s, cur_e))
                labels.append(r)
                cur_s, cur_e = a, b
        rows.append((cur_s, cur_e))
        labels.append(r)
    return (np.array(rows, dtype=np.float64).reshape(-1, 2), np.array(labels, dtype=np.int32), names)


def identity_table(names: Sequence, labels: Sequence[str]) -> np.ndarray:
    """reference label names (string order, ``reference_arrays``) and a file's hypothesis labels -> int32 (32,): for reference
    label r the index g of the hypothesis label equal to its name, else -1 (also for r >= len(names))"""
    index = {label: g for g, label in enumerate(labels)}
    out = np.full(MAX_REFERENCE_LABELS, -1, dtype=np.int32)
    for r, name in enumerate(names):
        out[r] = index.get(name, -1)
    return out


def pack_identities(references: Sequence[Annotation], regions: Optional[Sequence], labels: Sequence[Sequence[str]]) \
        -> np.ndarray:
    """per-file references, scored regions (or None) and hypothesis labels -> the table of dg_sweep_set_identities, int32
    (files, 32): each file's :func:`identity_table` of the reference's names after cropping to its regions"""
    return np.ascontiguousarray(np.stack([
        identity_table(reference_arrays(ref, None if regions is None else regions[f])[2], labels[f])
        for f, ref in enumerate(references)]), dtype=np.int32)


def _rate(num: np.ndarray, total: np.ndarray) -> np.ndarray:
    """num / total per trial, as a fraction; with total = 0: 0 when num is 0, else 1 (pyannote's ``compute_metric`` of both
    error rates)"""
    safe = np.where(total > 0, total, 1.0)
    return np.where(total > 0, num / safe, np.where(num > 0, 1.0, 0.0))


@dataclass
class DERComponents:
    """Diarization error rate components in seconds, one entry per trial (float64 (T,) each)."""
    false_alarm: np.ndarray
    missed_detection: np.ndarray
    confusion: np.ndarray
    correct: np.ndarray
    total: np.ndarray

    @classmethod
    def from_array(cls, comp: np.ndarray) -> "DERComponents":
        """float64 (T, 5) in dg_sweep_score's order {false alarm, missed detection, confusion, correct, total}"""
        comp = np.asarray(comp, dtype=np.float64).reshape(-1, 5)
        return cls(*(comp[:, i].copy() for i in range(5)))

    def as_array(self) -> np.ndarray:
        return np.stack([self.false_alarm, self.missed_detection, self.confusion, self.correct, self.total], axis=1)

    @property
    def der(self) -> np.ndarray:
        """(false alarm + missed detection + confusion) / total per trial (:func:`_rate`)"""
        return _rate(self.false_alarm + self.missed_detection + self.confusion, self.total)

    def __add__(self, other: "DERComponents") -> "DERComponents":
        """the components of several files summed per trial (the "TOTAL" row of pyannote's report)"""
        return DERComponents.from_array(self.as_array() + other.as_array())


@dataclass
class IdentificationErrorComponents(DERComponents):
    """Identification error rate components in seconds, one entry per trial: the fields of :class:`DERComponents`, the
    labels matched by name."""

    @property
    def ier(self) -> np.ndarray:
        """(false alarm + missed detection + confusion) / total per trial (:func:`_rate`)"""
        return _rate(self.false_alarm + self.missed_detection + self.confusion, self.total)

    def __add__(self, other: "IdentificationErrorComponents") -> "IdentificationErrorComponents":
        """the components of several files summed per trial"""
        return IdentificationErrorComponents.from_array(self.as_array() + other.as_array())


@dataclass
class SweepOutputs:
    header: np.ndarray        # int32 (T, N, 4)
    turns: np.ndarray         # uint32, n_turns valid
    n_turns: int
    out_start: np.ndarray     # (N,) per-chunk output start / resolution
    out_res: np.ndarray
    maps: Optional[torch.Tensor] = None      # int32 (T, N, K) on the device
    centers: Optional[torch.Tensor] = None   # float64 (T, M, D) on the device
    device_seconds: float = 0.0


_AUDIO_STREAMS = 3            # audio streams a network pass over several files uses in turn (see FileBatches)


def seg_resolution(config: SpeakerDiarizationConfig, start: float, F: int) -> float:
    """seconds per score frame of a window starting at ``start``: ``SpeakerDiarization.__call__``'s
    waveforms[0].extent.duration / F, the extent of a window of 1 / sample_rate frames"""
    sr = config.sample_rate
    end = start + int(np.rint(config.duration * sr)) * (1 / sr)
    return (end - start if end > start else 0.0) / F


def stream_plan(starts: np.ndarray, config: SpeakerDiarizationConfig, F: int):
    """The post-path plan of a fresh stream (empty history) whose chunks start at ``starts`` (N,), with F score frames per
    chunk -> contiguous (plan int32 (N, 4 + nw), out_start float64 (N,), out_res float64 (N,))"""
    starts = np.asarray(starts, dtype=np.float64)
    nw = int(round(config.latency / config.step))
    plans = post_plan(starts, seg_resolution(config, float(starts[0]), F), np.zeros(0), np.zeros(0), nw, F, config.step,
                      config.latency)
    return tuple(np.ascontiguousarray(a, dtype=t) for a, t in zip(plans, (np.int32, np.float64, np.float64)))


def dataset_plan(fws: Sequence[FileWindows], config: SpeakerDiarizationConfig, F: int):
    """The :func:`stream_plan` of each of several files, concatenated in file order.  post.cu finds chunk c's aggregated
    buffers at chunks c - (nb - 1) .. c with nb <= (c's index in its file) + 1, so no chunk reaches into the previous
    file."""
    parts = [stream_plan(fw.starts, config, F) for fw in fws]
    return tuple(np.ascontiguousarray(np.concatenate([p[i] for p in parts])) for i in range(3))


def trial_groups(num_trials: int, num_chunks: int) -> List[slice]:
    """consecutive slices of the trials, one per launch: at most TRIALS_PER_LAUNCH trials and TRIAL_CHUNKS_PER_LAUNCH
    trial-chunks each"""
    per = min(TRIALS_PER_LAUNCH, TRIAL_CHUNKS_PER_LAUNCH // num_chunks)
    if per < 1:
        raise ValueError(f"{num_chunks} chunks exceed the {TRIAL_CHUNKS_PER_LAUNCH} trial-chunks of one launch")
    return [slice(i, min(i + per, num_trials)) for i in range(0, num_trials, per)]


def pack_references(references: Sequence[Annotation], regions: Optional[Sequence] = None):
    """per-file references -> the reference arguments of dg_sweep_score_files: (rows float64 (S, 2), labels int32 (S,),
    row offsets int32 (files + 1,), label counts int32 (files,)); each file's rows as ``reference_arrays`` gives them, cropped
    to the file's entry of ``regions`` when given"""
    rows, labels, offsets, counts = [], [], [0], []
    for f, ref in enumerate(references):
        r, lab, names = reference_arrays(ref, None if regions is None else regions[f])
        rows.append(r)
        labels.append(lab)
        offsets.append(offsets[-1] + len(r))
        counts.append(len(names))
    return (np.ascontiguousarray(np.concatenate(rows), dtype=np.float64),
            np.ascontiguousarray(np.concatenate(labels), dtype=np.int32), np.array(offsets, dtype=np.int32),
            np.array(counts, dtype=np.int32))


def file_turns(header: np.ndarray, turns: np.ndarray, c0: int, c1: int):
    """header int32 (T, N, 4) and the packed turns of a sweep over several files -> the header (T, c1 - c0, 4) of the file
    with chunks [c0, c1) and its turns alone (offsets renumbered so that its blocks tile its turn list)"""
    h = np.ascontiguousarray(header[:, c0:c1])
    flat = h.reshape(-1, 4)
    cnt = flat[:, 1].astype(np.int64)
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)
    src = np.repeat(flat[:, 0].astype(np.int64) - start, cnt) + np.arange(int(cnt.sum()))
    flat[:, 0] = start
    own = turns[src]
    return h, own, len(own)


def parse_latencies(config, latencies: Iterable) -> Tuple[float, ...]:
    """the latencies a sweep over several latencies can score, ascending: ``latencies`` with ``config.latency`` added, each
    ``"min"`` (= step), ``"max"`` (= duration) or a number in [step, duration], else ValueError"""
    out = {float(config.latency)}
    for lat in latencies:
        value = config.step if lat == "min" else (config.duration if lat == "max" else lat)
        if isinstance(value, (bool, str)) or not isinstance(value, (int, float, np.integer, np.floating)) or \
                not config.step <= float(value) <= config.duration:
            raise ValueError(f"latency {lat!r}: need 'min', 'max' or a number in [step, duration] = "
                             f"[{config.step}, {config.duration}]")
        out.add(float(value))
    return tuple(sorted(out))


def latency_index(config, latencies: Sequence[float], latency) -> int:
    """the index of ``latency`` ("min" / "max" as in the configs) in ``latencies``, else ValueError"""
    value = config.step if latency == "min" else (config.duration if latency == "max" else latency)
    try:
        return list(latencies).index(float(value))
    except (TypeError, ValueError):
        raise ValueError(f"latency {latency!r} was not constructed (the sweep's latencies: {list(latencies)})") from None


def at_latency(config, latency: float):
    """a shallow copy of ``config`` with another latency (everything else, the models included, shared)"""
    out = copy.copy(config)
    out._latency = latency
    return out


class LatencyUnits:
    """The host plan of a dataset sweep over several latencies.

    ``latency`` enters a file's windows only through its padding (``get_file_padding``): right padding ``latency - step``
    and, for a file shorter than the chunk, left padding.  So the windows of a file at two latencies with the same left
    padding are a prefix of each other: the larger latency only appends windows at the end.  A *unit* is the windows of one
    file at the largest latency of a group with equal left padding (in samples); the network pass runs over units.  A file
    at least one chunk long has no left padding at any latency and is one unit; a shorter one has a unit per distinct left
    padding.

    One exception (``stream_form``, the fused diarization pass): :class:`FileBatches` cuts batches of 256 windows from window
    0, and the sinc front end runs in its stream form for batches of at least 4 windows and in its per-window form for
    smaller ones (``run_sinc_prep``, ``csrc/api_seg.cu``), which round differently.  A latency whose last batch holds 1 to
    3 windows would see them computed in a longer batch of its unit, so it gets a unit of its own (unless its windows are
    the unit's exactly).  Batches of 4 or more windows give every window the same bits whatever their length
    (``test_gpu_sweep_latencies``).  The VAD sweep's segmentation pass takes no hop hint, so always the per-window form.

    A *virtual file* is a (latency, file) pair: the first ``num_windows[l, f]`` chunks of unit ``unit_of[l, f]``, each with
    the plan row, output times and timestamp shift of that latency (:meth:`plan`, :meth:`tables`).  The clustering is causal
    and never reads the latency, so one clustering per unit and trial serves every latency the unit holds."""

    def __init__(self, waveforms: Sequence[np.ndarray], config, latencies: Iterable, stream_form: bool = True):
        self.config = config
        self.latencies = parse_latencies(config, latencies)
        self.nw = int(round(self.latencies[-1] / config.step))          # plan width: the largest latency's
        nl, nf = len(self.latencies), len(waveforms)
        self.unit_of = np.zeros((nl, nf), dtype=np.int64)
        self.num_windows = np.zeros((nl, nf), dtype=np.int64)
        self.starts: List[List[np.ndarray]] = [[None] * nf for _ in range(nl)]
        self.shifts = np.zeros((nl, nf), dtype=np.float64)
        self.unit_windows: List[FileWindows] = []
        for f, x in enumerate(waveforms):
            fws = [file_windows(x, at_latency(config, lat)) for lat in self.latencies]
            by_left: Dict[int, List[int]] = {}
            for li, fw in enumerate(fws):
                by_left.setdefault(int(np.rint(fw.padding[0] * config.sample_rate)) if fw.padding[0] > 0 else 0,
                                   []).append(li)
            groups: Dict[tuple, List[int]] = {}
            for n_left, lis in by_left.items():
                n_max = fws[lis[-1]].num_windows
                for li in lis:
                    n = fws[li].num_windows
                    apart = stream_form and n != n_max and 0 < n % NETWORK_BATCH < STREAM_FORM_MIN_BATCH
                    groups.setdefault((n_left, n if apart else -1), []).append(li)
            for lis in groups.values():
                unit = fws[lis[-1]]                                      # the group's largest latency
                for li in lis:
                    fw = fws[li]
                    n = fw.num_windows
                    if fw.offset != unit.offset or n > unit.num_windows or not np.array_equal(fw.starts, unit.starts[:n]) \
                            or not np.array_equal(fw.samples[:len(unit.samples)], unit.samples[:len(fw.samples)]):
                        raise AssertionError(f"file {f}: the windows at latency {self.latencies[li]} are not a prefix of "
                                             f"those at {self.latencies[lis[-1]]}")
                    self.unit_of[li, f] = len(self.unit_windows)
                    self.num_windows[li, f] = n
                    self.starts[li][f] = fw.starts
                    self.shifts[li, f] = -fw.padding[0]
                self.unit_windows.append(unit)
        self.unit_offsets = np.ascontiguousarray(np.cumsum([0] + [fw.num_windows for fw in self.unit_windows]),
                                                 dtype=np.int32)
        self._plans: Optional[List[tuple]] = None

    @property
    def num_chunks(self) -> int:
        """real chunks: the units' windows"""
        return int(self.unit_offsets[-1])

    def num_virtual(self, sel: Sequence[int]) -> int:
        """virtual chunks of the latencies with indices ``sel``"""
        return int(self.num_windows[list(sel)].sum())

    def plan(self, F: int):
        """computes each latency's plans for F score frames per chunk (once the network pass knows F) and drops the units'
        audio"""
        self.unit_windows = []
        self._plans = []
        for li, lat in enumerate(self.latencies):
            cfg = at_latency(self.config, lat)
            parts = [stream_plan(s, cfg, F) for s in self.starts[li]]
            plan = np.zeros((sum(len(p[0]) for p in parts), 4 + self.nw), dtype=np.int32)
            cat = np.concatenate([p[0] for p in parts])
            plan[:, :cat.shape[1]] = cat                               # zero-padded to the largest latency's width
            self._plans.append((plan, np.concatenate([p[1] for p in parts]), np.concatenate([p[2] for p in parts])))

    def tables(self, sel: Sequence[int]):
        """the virtual layout of the latencies with indices ``sel``, latency-major then file order -> (vchunk int32 (Nv,),
        virtual file offsets int32 (nvf + 1,), plan int32 (Nv, 4 + nw), out_start, out_res float64 (Nv,), shifts float64
        (nvf,)), all contiguous"""
        vchunk, counts = [], []
        for li in sel:
            for f in range(self.num_windows.shape[1]):
                n = int(self.num_windows[li, f])
                vchunk.append(self.unit_offsets[self.unit_of[li, f]] + np.arange(n))
                counts.append(n)
        return (np.ascontiguousarray(np.concatenate(vchunk), dtype=np.int32),
                np.ascontiguousarray(np.cumsum([0] + counts), dtype=np.int32),
                *(np.ascontiguousarray(np.concatenate([self._plans[li][i] for li in sel])) for i in range(3)),
                np.ascontiguousarray(self.shifts[list(sel)].reshape(-1)))


class FileBatches:
    """Iterates over the window batches of a network pass over several files, in file then batch order: each a dense
    (B, chunk_samples) device tensor of B <= 256 consecutive windows of one file.  Every batch holds windows of one file only,
    cut at the multiples of 256 from that file's window 0: the batch is the unit of the network pass's arithmetic (the sinc
    layer's stream form covers one batch), so each file's outputs are the bits a pass over it alone gives.  A file's audio
    is pushed as its batches need it; nothing drains or synchronises between files.

    Iterate under ``torch.cuda.device(device)`` and keep the object until the batches are consumed: it owns the audio
    streams, and destroying one frees device memory, which waits for the device."""

    def __init__(self, fws: Sequence[FileWindows], config, device: torch.device):
        self.fws, self.config, self.device = fws, config, device
        self.streams: List[DeviceAudioStream] = []

    def __iter__(self):
        cfg, streams = self.config, self.streams
        for i, fw in enumerate(self.fws):
            # a few streams in turn: a reset waits for the uploads of its stream, so reuse the one whose file was
            # submitted longest ago (its batches have left the consumer's pipeline)
            if len(streams) < _AUDIO_STREAMS:
                streams.append(DeviceAudioStream(cfg.duration, cfg.step, cfg.sample_rate, max_windows=NETWORK_BATCH,
                                                 device=self.device))
            stream = streams[i % _AUDIO_STREAMS]
            if i >= _AUDIO_STREAMS:
                stream.reset()
            pushed = fw.offset
            for i0 in range(0, fw.num_windows, NETWORK_BATCH):
                B = min(NETWORK_BATCH, fw.num_windows - i0)
                need = fw.offset + (i0 + B - 1) * fw.step_samples + fw.chunk_samples
                stream.push(fw.samples[pushed:need])
                pushed = need
                yield stream.windows(B)


def _indexed(device: torch.device) -> torch.device:
    """``device`` with an index: "cuda" alone is the current device"""
    return device if device.index is not None else torch.device("cuda", torch.cuda.current_device())


def _timed(device: torch.device, call):
    """Runs ``call(cuda_stream)``, one C entry point that enqueues on the current stream of ``device``, between two CUDA
    events -> (its status, seconds).  ``seconds()`` waits for the second event and returns the device time between the
    two: for the caller to ask once it has checked the status."""
    with torch.cuda.device(device):
        st = torch.cuda.current_stream(device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        rc = call(st.cuda_stream)
        e1.record(st)

    def seconds() -> float:
        e1.synchronize()
        return e0.elapsed_time(e1) / 1e3
    return rc, seconds


def _set_regions(setter, handle, regions: Optional[tuple]):
    """``setter`` (dg_sweep_set_scored_regions / dg_vad_sweep_set_scored_regions): the handle's scored regions for its next
    scoring calls, ``pack_regions``' (rows, offsets), or none (None: the hypotheses are scored whole)"""
    if regions is None:
        _lib.check(setter(handle, 0, None, None))
    else:
        rows, offsets = regions
        _lib.check(setter(handle, len(offsets) - 1, rows.ctypes.data, offsets.ctypes.data))


def _turn_list_call(owner, device: torch.device, guess: int, call) -> Tuple[int, float]:
    """Runs ``call(turns, capacity, n, cuda_stream)``, the last four arguments of an entry point that downloads a packed
    turn list, into ``owner._turns`` (uint32, grown to ``guess`` entries first) -> (turns written, device seconds of the
    call).  An entry point that finds more turns than the buffer holds reports how many: the buffer grows to that and the
    call runs once more (its seconds are the ones returned)."""
    if len(owner._turns) < guess:
        owner._turns = np.empty(guess, dtype=np.uint32)
    n = C.c_int()
    for attempt in range(2):
        rc, seconds = _timed(device, lambda st: call(owner._turns.ctypes.data, len(owner._turns), C.byref(n), st))
        if rc == -1 and n.value > len(owner._turns):
            owner._turns = np.empty(n.value, dtype=np.uint32)
            continue
        _lib.check(rc)
        break
    return n.value, seconds()


class HyperParameterSweep:
    """Runs ``SpeakerDiarization(config)`` over a file for many (tau_active, rho_update, delta_new) trials at the cost of one
    network pass.  Needs the native segmentation and embedding models.

        sweep = HyperParameterSweep(config)
        predictions = sweep.run(waveform, uri="file1", trials=[{"tau_active": 0.5}, {"delta_new": 0.8, "rho_update": 0.2}])
    """

    def __init__(self, config: SpeakerDiarizationConfig):
        self.config = config
        self.pipeline = SpeakerDiarization(config)
        if self.pipeline._native_models() is None:
            raise _lib.DiartB200Error("HyperParameterSweep needs the native segmentation and embedding models")
        self.device = _indexed(self.pipeline.segmentation.device)
        self._h: Optional[C.c_void_p] = None
        self._dims = None
        self._turns = np.empty(0, dtype=np.uint32)
        self.timing: Dict[str, float] = {}        # seconds of the last run: network, sweep (device events), assembly

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                _lib.lib().dg_sweep_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    # ------------------------------------------------------------------ network pass
    def network_pass(self, fw: FileWindows):
        """scores (N, F, K) and embeddings (N, K, D) of every window, on the device: the fused pipeline in batches of 256
        (its own clustering runs too; its maps are not used)"""
        return self.network_pass_files([fw])

    def network_pass_files(self, fws: Sequence[FileWindows]):
        """:meth:`network_pass` of several files as one pipelined flow -> their scores and embeddings concatenated in file
        order, each file's the bits :meth:`network_pass` gives for it alone (:class:`FileBatches`).  Two batches are in
        flight at a time; nothing drains or synchronises between files."""
        pipe = self.pipeline
        pipe.reset()
        batches = FileBatches(fws, self.config, self.device)
        segs, embs, inflight = [], [], []

        def collect():
            seg, emb, _ = pipe.collect()
            segs.append(seg)
            embs.append(emb)
            inflight.pop(0)

        with torch.cuda.device(self.device):
            for windows in batches:
                inflight.append(windows)                      # must stay alive until collected
                pipe.submit(windows)
                if len(inflight) == 2:
                    collect()
            while inflight:
                collect()
            return torch.cat(segs), torch.cat(embs)

    def network_pass_sets(self, fws: Sequence[FileWindows], sets: Sequence[Tuple[float, float, bool]]):
        """:meth:`network_pass_files` for several OSP sets (:func:`osp_sets`) -> scores (N, F, K) and the embeddings of
        every set (G, N, K, D), set g's the bits :meth:`network_pass_files` gives under a config with that set.  One
        ``dg_pipeline_nets_sets`` per batch writes into the two tensors; consecutive batches run on two streams in turn, so
        two are in flight."""
        pipe = self.pipeline
        pipe.reset()
        h, F, K, D = pipe._ensure_fused(fws[0].chunk_samples)
        N, G = sum(fw.num_windows for fw in fws), len(sets)
        osp = np.ascontiguousarray([s[:2] for s in sets], dtype=np.float32)
        normalize = np.ascontiguousarray([int(s[2]) for s in sets], dtype=np.int32)
        seg = torch.empty((N, F, K), device=self.device)
        embs = torch.empty((G, N, K, D), device=self.device)
        batches = FileBatches(fws, self.config, self.device)
        with torch.cuda.device(self.device):
            current = torch.cuda.current_stream(self.device)
            lanes = [torch.cuda.Stream(self.device), torch.cuda.Stream(self.device)]
            inflight, n0 = [], 0
            for i, windows in enumerate(batches):
                lane = lanes[i % 2]
                lane.wait_stream(current)
                B = windows.shape[0]
                _lib.check(_lib.lib().dg_pipeline_nets_sets(h, windows.data_ptr(), B, windows.shape[1], G, osp.ctypes.data,
                                                            normalize.ctypes.data, seg[n0].data_ptr(), embs[0, n0].data_ptr(),
                                                            N * K * D, lane.cuda_stream))
                n0 += B
                inflight.append((windows, lane))             # the windows must stay alive until their lane is waited for
                if len(inflight) == 2:
                    current.wait_stream(inflight.pop(0)[1])
            while inflight:
                current.wait_stream(inflight.pop(0)[1])
        return seg, embs

    # ------------------------------------------------------------------ clustering + post-path for T trials
    def _handle(self, F: int, K: int, D: int, nw: Optional[int] = None):
        """the dg_sweep handle for these dimensions; ``nw``: its plan width, by default the config's latency / step"""
        if nw is None:
            nw = int(round(self.config.latency / self.config.step))
        dims = (F, K, D, nw)
        if self._h is None or self._dims != dims:
            if self._h is not None:
                _lib.lib().dg_sweep_destroy(self._h)
                self._h = None
            ham = np.ascontiguousarray(np.hamming(F), dtype=np.float64)
            h = C.c_void_p()
            _lib.check(_lib.lib().dg_sweep_create(int(self.config.max_speakers), D, F, K, nw, ham.ctypes.data,
                                                  self.device.index, C.byref(h)))
            self._h, self._dims = h, dims
        return self._h, nw

    def _run_trials(self, entry, file_args: tuple, lead: tuple, seg: torch.Tensor, emb: torch.Tensor, plans,
                    params: np.ndarray, keep_state: bool, trial_sets: Optional[Tuple[int, np.ndarray]] = None,
                    seeds: Optional[Tuple[np.ndarray, np.ndarray]] = None) -> SweepOutputs:
        """The body of :meth:`sweep` and :meth:`DatasetSweep.sweep`.  ``entry``: dg_sweep_run, or dg_sweep_run_files with
        ``file_args`` = what it takes after the chunk count (files, chunk offsets) and ``lead`` = (files,), the leading
        dimension of its centroids.  ``plans``: (plan, out_start, out_res) of the N chunks.  ``trial_sets``: (G, set of each
        trial) with ``emb`` (G, N, K, D), or None with ``emb`` (N, K, D).  ``seeds``: the files' known centroids
        (:func:`_set_seeds`), or None."""
        N, F, K = seg.shape
        D, M = emb.shape[-1], int(self.config.max_speakers)
        h, _ = self._handle(F, K, D)
        _set_trial_sets(h, trial_sets)
        _set_seeds(h, seeds)
        plan, out_start, out_res = plans
        params = np.ascontiguousarray(params, dtype=np.float64)
        T = len(params)
        header = np.empty((T, N, 4), dtype=np.int32)
        maps = torch.empty((T, N, K), dtype=torch.int32, device=self.device) if keep_state else None
        centers = torch.empty((*lead, T, M, D), dtype=torch.float64, device=self.device) if keep_state else None
        n_turns, seconds = _turn_list_call(self, self.device, T * N * 8, lambda *turn_list: entry(
            h, seg.data_ptr(), emb.data_ptr(), N, *file_args, params.ctypes.data, T, plan.ctypes.data, _lib.ptr(maps),
            _lib.ptr(centers), header.ctypes.data, *turn_list))
        return SweepOutputs(header, self._turns[:n_turns].copy(), n_turns, out_start, out_res, maps, centers, seconds)

    def _score_trials(self, entry, file_args: tuple, lead: tuple, seg: torch.Tensor, emb: torch.Tensor, plans,
                      params: np.ndarray, shift, reference: tuple, segments: bool = False, regions: Optional[tuple] = None,
                      trial_sets: Optional[Tuple[int, np.ndarray]] = None,
                      seeds: Optional[Tuple[np.ndarray, np.ndarray]] = None, identities: Optional[np.ndarray] = None):
        """The body of :meth:`sweep_score` and of each launch of :meth:`DatasetSweep.score` -> (components ``lead`` +
        (T, 5), device seconds, hypothesis offsets, hypothesis segments).  ``entry``: dg_sweep_score, or
        dg_sweep_score_files with ``file_args`` and ``lead`` as in :meth:`_run_trials`.  ``shift``: the timestamp shift, or
        the address of the per-file shifts.  ``reference``: the entry point's four reference arguments (rows, labels,
        then the row and label counts, or the addresses of the per-file row offsets and label counts).  ``segments`` is
        for the one-file entry point.  ``regions``: ``pack_regions`` of the files' scored regions, or None.  ``trial_sets``
        and ``seeds`` as in :meth:`_run_trials`.  ``identities``: :func:`pack_identities`' table to score the identification
        error rate, or None (DER)."""
        N, F, K = seg.shape
        h, _ = self._handle(F, K, emb.shape[-1])
        _set_regions(_lib.lib().dg_sweep_set_scored_regions, h, regions)
        _set_trial_sets(h, trial_sets)
        _set_seeds(h, seeds)
        _set_identities(h, identities)
        plan, out_start, out_res = plans
        params = np.ascontiguousarray(params, dtype=np.float64)
        T, M = len(params), int(self.config.max_speakers)
        comp = np.empty((*lead, T, 5), dtype=np.float64)
        offsets = hseg = None
        if segments:
            offsets = torch.empty(T * M + 1, dtype=torch.int32, device=self.device)
            hseg = torch.empty((T * N * 8, 2), dtype=torch.float64, device=self.device)
        rc, seconds = _timed(self.device, lambda st: entry(
            h, seg.data_ptr(), emb.data_ptr(), N, *file_args, params.ctypes.data, T, plan.ctypes.data, out_start.ctypes.data,
            out_res.ctypes.data, shift, PATCH_COLLAR, *reference, comp.ctypes.data, _lib.ptr(offsets), _lib.ptr(hseg),
            0 if hseg is None else hseg.shape[0], st))
        _lib.check(rc)
        secs = seconds()
        if segments:
            hseg = hseg[:int(offsets[-1])]
        return comp, secs, offsets, hseg

    def sweep(self, seg: torch.Tensor, emb: torch.Tensor, starts: np.ndarray, params: np.ndarray,
              keep_state: bool = False, trial_sets: Optional[Tuple[int, np.ndarray]] = None) -> SweepOutputs:
        """dg_sweep_run over device scores / embeddings of N chunks starting at ``starts`` for params (T, 3); ``trial_sets``
        as in :meth:`_run_trials`"""
        plans = stream_plan(starts, self.config, seg.shape[1])
        return self._run_trials(_lib.lib().dg_sweep_run, (), (), seg, emb, plans, params, keep_state, trial_sets)

    def sweep_score(self, seg: torch.Tensor, emb: torch.Tensor, fw: FileWindows, params: np.ndarray, ref_rows: np.ndarray,
                    ref_labels: np.ndarray, num_ref_labels: int, segments: bool = False, regions: Optional[tuple] = None,
                    trial_sets: Optional[Tuple[int, np.ndarray]] = None):
        """dg_sweep_score over device scores / embeddings of ``fw``'s chunks for params (T, 3) against a reference in
        ``reference_arrays`` form -> (components (T, 5), device seconds, hypothesis offsets, hypothesis segments).  The last
        two are device tensors when ``segments`` (int32 (T * max_speakers + 1,) and float64 (n, 2), see the C header), else
        None; the hypothesis segments are the uncropped predictions.  ``regions``: ``pack_regions([scored regions])`` to
        crop the hypotheses to (the reference rows cropped alike), or None."""
        rows = np.ascontiguousarray(ref_rows, dtype=np.float64)
        labels = np.ascontiguousarray(ref_labels, dtype=np.int32)
        reference = (rows.ctypes.data, labels.ctypes.data, len(rows), int(num_ref_labels))
        plans = stream_plan(fw.starts, self.config, seg.shape[1])
        return self._score_trials(_lib.lib().dg_sweep_score, (), (), seg, emb, plans, params, -fw.padding[0], reference,
                                  segments, regions, trial_sets)

    def _network_pass_trials(self, fw: FileWindows, trials: Sequence[Mapping[str, float]]):
        """the network pass of one file for trials that may carry OSP sets -> (params (T, 3), scores, embeddings, set of each
        trial): without other sets than the config's :meth:`network_pass` and no trial sets, else :meth:`network_pass_sets`
        over the distinct sets the trials name"""
        sets = trial_osp_sets(self.config, trials)
        index, params = trial_osp_params(trials, self.config, sets)
        if len(sets) == 1:
            seg, emb = self.network_pass(fw)
            return params, seg, emb, None
        seg, embs = self.network_pass_sets([fw], sets)
        return params, seg, embs, (len(sets), index)

    def _seg_resolution(self, start: float, F: int) -> float:
        return seg_resolution(self.config, start, F)

    # ------------------------------------------------------------------ the public entry
    def run(self, waveform: np.ndarray, uri: Optional[str] = None,
            trials: Sequence[Mapping[str, float]] = ({},)) -> List[Annotation]:
        """1-D float32 waveform at ``config.sample_rate`` -> one whole-file prediction per trial (the prediction
        ``Benchmark.run_single`` returns for a pipeline with that trial's tau_active / rho_update / delta_new).  A trial may
        also carry ``gamma``, ``beta`` and ``normalize_embedding_weights``: the network pass then computes the embeddings of
        every distinct such set once (:meth:`network_pass_sets`)."""
        trial_osp_params(trials, self.config, trial_osp_sets(self.config, trials))    # bad trials fail before the networks
        t0 = time.perf_counter()
        fw = file_windows(waveform, self.config)
        params, seg, emb, sets = self._network_pass_trials(fw, trials)
        torch.cuda.synchronize(self.device)
        t1 = time.perf_counter()
        labels = [f"speaker{g}" for g in range(int(self.config.max_speakers))]
        shift = -fw.padding[0]
        out, dev, host = [], 0.0, 0.0
        for i in range(0, len(params), TRIALS_PER_LAUNCH):
            part = None if sets is None else (sets[0], sets[1][i:i + TRIALS_PER_LAUNCH])
            r = self.sweep(seg, emb, fw.starts, params[i:i + TRIALS_PER_LAUNCH], trial_sets=part)
            dev += r.device_seconds
            t2 = time.perf_counter()
            out += assemble_predictions(r.header, r.turns, r.n_turns, r.out_start, r.out_res, labels, shift, uri)
            host += time.perf_counter() - t2
        self.timing = {"network": t1 - t0, "sweep": dev, "assembly": host}
        return out

    def score(self, waveform: np.ndarray, reference: Annotation, trials: Sequence[Mapping[str, float]] = ({},),
              metric=None, uem=None) -> DERComponents:
        """1-D float32 waveform at ``config.sample_rate`` and its reference annotation -> the diarization error rate
        components of every trial's whole-file prediction (the one :meth:`run` returns) against the reference.  One network
        pass, one ``dg_sweep_score`` per 1024 trials; no annotation is built.  At most 32 reference labels.

        ``metric``: a :class:`DiarizationErrorRate` (or pyannote.metrics' own) with a forgiveness collar and / or
        ``skip_overlap``; None is ``DiarizationErrorRate()``.  ``uem``: the scored parts of the file, ``(start, end)`` pairs
        or ``Segment``s in the reference's time base; None scores everything (DESIGN.md "DER scoring").  Trials may carry OSP
        sets as in :meth:`run`."""
        trial_osp_params(trials, self.config, trial_osp_sets(self.config, trials))
        collar, skip_overlap = metric_protocol(metric, "DiarizationErrorRate")
        uem = check_uem(uem)
        regions = None
        if collar > 0 or skip_overlap or uem is not None:
            regions = scored_regions(reference, collar, skip_overlap, uem)
        rows, labels, names = reference_arrays(reference, regions)
        t0 = time.perf_counter()
        fw = file_windows(waveform, self.config)
        params, seg, emb, sets = self._network_pass_trials(fw, trials)
        torch.cuda.synchronize(self.device)
        t1 = time.perf_counter()
        comps, dev = [], 0.0
        for i in range(0, len(params), TRIALS_PER_LAUNCH):
            part = None if sets is None else (sets[0], sets[1][i:i + TRIALS_PER_LAUNCH])
            comp, secs, _, _ = self.sweep_score(seg, emb, fw, params[i:i + TRIALS_PER_LAUNCH], rows, labels, len(names),
                                                regions=None if regions is None else pack_regions([regions]), trial_sets=part)
            comps.append(comp)
            dev += secs
        self.timing = {"network": t1 - t0, "score": dev}
        return DERComponents.from_array(np.concatenate(comps))

    def score_files(self, files: Iterable[Tuple[np.ndarray, Annotation]], trials: Sequence[Mapping[str, float]] = ({},),
                    metric=None) -> Tuple[List[DERComponents], DERComponents]:
        """``files``: (waveform, reference) pairs -> (components per file, their sum).  ``total.der`` per trial is the
        value the reference's ``Optimizer.objective`` minimises over a dataset (a fraction, not a percentage).  Runs as a
        :class:`DatasetSweep` over the files, built with the OSP sets the trials name.  ``metric`` as in :meth:`score`."""
        metric_protocol(metric, "DiarizationErrorRate")        # a bad metric fails before the network pass
        sets = trial_osp_sets(self.config, trials)
        dataset = DatasetSweep(self.config, [(None, waveform, reference) for waveform, reference in files], sweep=self,
                               osp=[osp_dict(s) for s in sets[1:]])
        out = dataset.score(trials, metric)
        self.timing = dict(dataset.timing)
        return out


class _DatasetSweep:
    """What the dataset sweeps share: the checks of the files, the chunk offsets, post-path plans and timestamp shifts of
    the concatenated files, the network pass a subclass runs once and keeps on the device (``_open``, ``_networks``), the
    packed references (``_pack_references``) and the loops of ``run`` and ``score`` over trial groups and files
    (``_score_group``, ``_components``)."""

    _pack_references = None   # staticmethod of the subclass: (references, regions) -> the reference arguments of its scoring entry
    _stream_form = True       # the network pass runs the sinc front end's stream form (LatencyUnits)
    _metric = ""              # the class name of the metric the subclass scores (metric_protocol)

    def __init__(self, config, files: Iterable[Tuple[Optional[str], np.ndarray, Optional[Annotation]]],
                 latencies: Optional[Iterable] = None, uems: Optional[Sequence] = None):
        files = list(files)
        if not files:
            raise ValueError("at least one file is needed")
        for i, (uri, x, _) in enumerate(files):
            if np.asarray(x).size == 0:
                raise ValueError(f"file {i} ({uri}) has no samples, so no windows")
        if uems is not None and (not isinstance(uems, (list, tuple)) or len(uems) != len(files)):
            raise ValueError(f"uems: need one entry (a uem or None) per file, {len(files)} in all")
        self.uems = [check_uem(u) for u in uems] if uems is not None else [None] * len(files)
        self.config = config
        self.uris = [uri for uri, _, _ in files]
        self.references = [ref for _, _, ref in files]
        self.units: Optional[LatencyUnits] = None
        if latencies is None:
            fws = [file_windows(x, config) for _, x, _ in files]   # (the padded audio is dropped after the network pass)
            self.offsets = np.ascontiguousarray(np.cumsum([0] + [fw.num_windows for fw in fws]), dtype=np.int32)
            trial_groups(1, self.num_chunks)                        # a dataset too large for one launch fails here
        else:
            # the network pass runs over the units; self.offsets are theirs
            self.units = LatencyUnits([x for _, x, _ in files], config, latencies, self._stream_form)
            fws = self.units.unit_windows
            self.offsets = self.units.unit_offsets
            trial_groups(1, max(self.units.num_virtual(range(len(self.units.latencies))), self.units.num_chunks))
        self.device = self._open()
        t0 = time.perf_counter()
        self._networks(fws)
        torch.cuda.synchronize(self.device)
        self.timing: Dict[str, float] = {"network": time.perf_counter() - t0}
        self._packs: Dict[tuple, tuple] = {}
        if self.units is not None:
            self.units.plan(self.seg.shape[1])
            self.plan = self.out_start = self.out_res = self.shifts = None
            self._virtual: Dict[tuple, tuple] = {}
            return
        self.plan, self.out_start, self.out_res = dataset_plan(fws, config, self.seg.shape[1])
        self.shifts = np.ascontiguousarray([-fw.padding[0] for fw in fws], dtype=np.float64)

    def _open(self) -> torch.device:
        """makes the pipeline whose networks run (an error if they are not native) -> their device"""
        raise NotImplementedError

    def _networks(self, fws: Sequence[FileWindows]):
        """runs the networks over every window of every file and keeps their outputs on the device, the scores as
        ``self.seg`` (N, F, K)"""
        raise NotImplementedError

    def _score_group(self, params: np.ndarray, refs: tuple, regions: Optional[tuple]) -> Tuple[np.ndarray, float]:
        """one scoring launch for one trial group against the packed references ``refs``, the hypotheses cropped to
        ``regions`` (``pack_regions``, or None) -> (components (files, T, width), device seconds)"""
        raise NotImplementedError

    def _components(self, f: int, comp: np.ndarray, refs: tuple):
        """file f's components object from its (T, width) slice of the launches' components; ``refs``: the packed
        references f indexes (a virtual file's in the sweeps over several latencies)"""
        raise NotImplementedError

    def _metric_kind(self, metric) -> Tuple[str, float, bool]:
        """``metric`` -> (the class name it scores, collar, skip_overlap); anything this sweep does not score: ValueError"""
        return (self._metric, *metric_protocol(metric, self._metric))

    def _pack(self, kind: str, references: List[Annotation], regions: Optional[list], copies: int) -> tuple:
        """the reference arguments of the scoring entry for metric class ``kind`` (files ``copies`` times)"""
        return self._pack_references(references, regions)

    def _packed(self, metric, copies: int = 1) -> Tuple[tuple, Optional[tuple]]:
        """the packed references (``_pack``) and scored regions (``pack_regions``, or None where nothing is cropped) of
        ``metric`` (:meth:`_metric_kind`) with the files' uems, every file ``copies`` times (latency-major), kept per (copies,
        metric kind, collar, skip_overlap) for later calls.  ``regions_seconds``: host seconds spent packing (about 0 when
        kept)."""
        kind, *protocol = self._metric_kind(metric)
        protocol = tuple(protocol)
        self._check_references()
        key = (copies, kind, *protocol)
        t0 = time.perf_counter()
        if key not in self._packs:
            regions = None
            if protocol != (0.0, False) or any(u is not None for u in self.uems):
                regions = [scored_regions(ref, *protocol, uem) for ref, uem in zip(self.references, self.uems)] * copies
            self._packs[key] = (self._pack(kind, self.references * copies, regions, copies),
                                None if regions is None else pack_regions(regions))
        self.regions_seconds = time.perf_counter() - t0
        return self._packs[key]

    @property
    def num_chunks(self) -> int:
        return int(self.offsets[-1])

    def _run(self, params: np.ndarray, launch, labels: Sequence[Sequence[str]]) -> List[List[Annotation]]:
        """``launch``: the trials of one group -> their :class:`SweepOutputs` over the concatenated chunks.  -> predictions
        [file][trial], each file's assembled from its own chunks and turns with its own speaker labels ``labels[f]``"""
        out: List[List[Annotation]] = [[] for _ in self.uris]
        dev = 0.0
        for g in trial_groups(len(params), self.num_chunks):
            r = launch(params[g])
            dev += r.device_seconds
            for f in range(len(self.uris)):
                c0, c1 = int(self.offsets[f]), int(self.offsets[f + 1])
                header, turns, n = file_turns(r.header, r.turns, c0, c1)
                out[f] += assemble_predictions(header, turns, n, self.out_start[c0:c1], self.out_res[c0:c1], labels[f],
                                               float(self.shifts[f]), self.uris[f])
        self.timing["sweep"] = dev
        return out

    def _score(self, params: np.ndarray, metric=None):
        """-> (components per file, their sum in file order) under ``metric``, one ``_score_group`` per trial group"""
        refs, regions = self._packed(metric)
        parts, dev = [], 0.0
        for g in trial_groups(len(params), self.num_chunks):
            part, secs = self._score_group(params[g], refs, regions)
            parts.append(part)
            dev += secs
        self.timing["score"] = dev
        comp = np.concatenate(parts, axis=1)
        per_file = [self._components(f, comp[f], refs) for f in range(len(self.uris))]
        return per_file, functools.reduce(operator.add, per_file)

    # ------------------------------------------------------------------ several latencies (built with ``latencies``)
    @property
    def latencies(self) -> Tuple[float, ...]:
        """the latencies the sweep can score, ascending"""
        return self.units.latencies if self.units is not None else (float(self.config.latency),)

    def _selection(self, latencies) -> List[int]:
        """the indices in :attr:`latencies` of the requested ones (None: all), ascending; ValueError for a latency that was
        not constructed"""
        if latencies is None:
            return list(range(len(self.latencies)))
        return sorted({latency_index(self.config, self.latencies, lat) for lat in latencies})

    def _chunk_range(self, f: int, latency) -> Tuple[int, int]:
        """the resident chunks [c0, c1) of file f's windows at ``latency`` (None: the config's)"""
        li = self._selection([self.config.latency if latency is None else latency])[0]
        if self.units is None:
            return int(self.offsets[f]), int(self.offsets[f + 1])
        c0 = int(self.units.unit_offsets[self.units.unit_of[li, f]])
        return c0, c0 + int(self.units.num_windows[li, f])

    def _tables(self, sel: Sequence[int]) -> tuple:
        """``LatencyUnits.tables`` of a selection, kept for later calls (the C calls read them by address)"""
        key = tuple(sel)
        if key not in self._virtual:
            self._virtual[key] = self.units.tables(key)
        return self._virtual[key]

    def _launched(self, sel: List[int]) -> List[int]:
        """the latencies whose virtual files a call for ``sel`` launches over"""
        return sel

    def _group_chunks(self, tabs: tuple) -> int:
        """the chunk count :func:`trial_groups` bounds for a launch over the virtual layout ``tabs``: its virtual chunks
        (header, turns), or the real chunks where more (the clustering's maps are [T][real chunks][K])"""
        return max(len(tabs[0]), self.units.num_chunks)

    def _run_latencies(self, params: np.ndarray, sel: List[int], launch, labels: Sequence[Sequence[str]]):
        """``launch(params, tables)``: the trials of one group -> their :class:`SweepOutputs` over the virtual chunks of
        ``tables``.  -> {latency: predictions [file][trial]}, each virtual file's assembled from its own chunks and turns with
        its file's speaker labels ``labels[f]``"""
        run = self._launched(sel)
        tabs = self._tables(run)
        vchunk, voff, _, out_start, out_res, shifts = tabs
        nf = len(self.uris)
        out = {self.latencies[li]: [[] for _ in self.uris] for li in sel}
        dev = 0.0
        for g in trial_groups(len(params), self._group_chunks(tabs)):
            r = launch(params[g], tabs)
            dev += r.device_seconds
            for k, li in enumerate(run):
                if li not in sel:
                    continue
                for f in range(nf):
                    v = k * nf + f
                    c0, c1 = int(voff[v]), int(voff[v + 1])
                    header, turns, n = file_turns(r.header, r.turns, c0, c1)
                    out[self.latencies[li]][f] += assemble_predictions(header, turns, n, out_start[c0:c1], out_res[c0:c1],
                                                                       labels[f], float(shifts[v]), self.uris[f])
        self.timing["sweep"] = dev
        return out

    def _score_latencies(self, params: np.ndarray, sel: List[int], launch, metric=None):
        """``launch(params, tables, references, regions)``: one scoring launch for the trials of one group -> (components
        (virtual files, T, width), device seconds).  -> {latency: (components per file, their sum in file order)} under
        ``metric``"""
        run = self._launched(sel)
        tabs = self._tables(run)
        nf, n = len(self.uris), len(run)
        refs, regions = self._packed(metric, n)            # every file's reference and regions once per latency
        parts, dev = [], 0.0
        for g in trial_groups(len(params), self._group_chunks(tabs)):
            part, secs = launch(params[g], tabs, refs, regions)
            parts.append(part)
            dev += secs
        self.timing["score"] = dev
        comp = np.concatenate(parts, axis=1)
        out = {}
        for k, li in enumerate(run):
            if li in sel:
                per_file = [self._components(k * nf + f, comp[k * nf + f], refs) for f in range(nf)]
                out[self.latencies[li]] = (per_file, functools.reduce(operator.add, per_file))
        return out

    def _check_references(self):
        missing = [self.uris[i] if self.uris[i] is not None else i for i, r in enumerate(self.references) if r is None]
        if missing:
            raise ValueError(f"files without a reference cannot be scored: {missing}")

    def _layout(self, tabs: tuple) -> tuple:
        """the layout arguments of the ``_latencies`` entry points after the device outputs: real chunks, units, unit offsets,
        virtual chunks, virtual files, virtual chunk table, virtual file offsets"""
        vchunk, voff = tabs[:2]
        u = self.units
        return (u.num_chunks, len(u.unit_offsets) - 1, u.unit_offsets.ctypes.data, len(vchunk), len(voff) - 1,
                vchunk.ctypes.data, voff.ctypes.data)


class DatasetSweep(_DatasetSweep):
    """A sweep over a whole dataset with the network outputs of every file kept on the device.

        ds = DatasetSweep(config, [("file1", waveform1, reference1), ("file2", waveform2, reference2)])
        per_file, total = ds.score([{"tau_active": 0.5}, {"delta_new": 0.8, "rho_update": 0.2}])
        best = int(np.argmin(total.der))

    ``files``: (uri, 1-D float32 waveform at ``config.sample_rate``, reference annotation or None).  The constructor runs
    the network pass of all files as one pipelined flow (:meth:`HyperParameterSweep.network_pass_files`) and keeps the
    concatenated scores and embeddings on the device: F K + K D float32 per chunk (3 516 + 6 144 B = 9.66 kB at the
    default models, F = 293 frames, K = 3 local speakers, D = 512; two chunks per second of audio at step 0.5 s, so about
    0.7 GB per 10 hours).  Then :meth:`score` and :meth:`run` cluster, post-process and score every (file, trial) pair in
    one launch per kernel and per trial group (at most 1024 trials and 4 Mi trial-chunks each) and run no network kernel:
    a tuning loop pays for the networks once.  For every file and trial the results are the bits a
    :class:`HyperParameterSweep` of that file alone gives, whatever the other files and their order.
    ``sweep``: a :class:`HyperParameterSweep` of the same config whose pipeline and handles to use (default: a new one).

    ``latencies``: the latencies the sweep can score besides ``config.latency`` (each ``"min"``, ``"max"`` or in [step,
    duration]).  The network pass then runs over units (:class:`LatencyUnits`: a file at least one chunk long is one unit,
    its windows at the largest latency, except for a latency whose last network batch holds 1 to 3 windows).
    :meth:`score_latencies` / :meth:`run_latencies` cluster every (unit, trial) once and run the post-path and scoring
    over every (latency, file) pair, in one launch per kernel and trial group whatever the number of latencies; for
    every latency L the results are the bits ``DatasetSweep`` built at latency L gives.  :meth:`score` / :meth:`run`
    return the ``config.latency`` entry.

    ``uems``: per file its uem (``(start, end)`` pairs or ``Segment``s in the reference's time base) or None, for every
    scoring call.  ``score`` and ``score_latencies`` take a ``metric`` (:class:`DiarizationErrorRate`, or
    pyannote.metrics' own) with a forgiveness collar and / or ``skip_overlap``; the default is ``DiarizationErrorRate()``.
    The packed references and scored regions are kept per metric.

    ``osp``: OSP sets besides the config's own, each a dict with any of ``gamma``, ``beta`` and
    ``normalize_embedding_weights`` (a missing key takes the config's value; equal float32 values collapse).  The network pass
    then computes the scores once and the embeddings of every set (``osp_sets`` lists them, the config's first; ``embs`` is
    (G, N, K, D), ``emb`` set 0), at (F K + G K D) float32 per chunk.  Trials of every method may carry those three keys, and
    each is clustered over its own set's embeddings in the same launches as the others: for every set the results are the
    bits a ``DatasetSweep`` whose config has that set's values gives.  A trial whose set was not constructed raises
    ValueError before any launch.  Without ``osp`` (or with only the config's set) the sweep runs as before.

    ``speakers``: known speakers (:class:`~diart_b200.speakers.KnownSpeakers`), one for every file or a sequence with one
    entry (a ``KnownSpeakers`` or None) per file; an empty one is None.  Every (file, trial) clustering then starts from the
    file's centroids, and file f's global speaker g is labelled ``labels[f][g]`` (``speaker_labels``): for every file and
    trial the results are those of ``SpeakerDiarization`` with ``set_known_speakers`` at that trial's values.  The latency
    units of a file and every OSP set take the file's seeds.  A wrong length or type, another dimension than the
    embeddings' or more than ``max_speakers`` speakers raises ValueError naming the file, before the network pass.
    ``score`` and ``score_latencies`` also take an :class:`IdentificationErrorRate` (or pyannote.metrics' own, unit weights):
    each reference label is matched to the hypothesis label of the same name, and the components come back as
    :class:`IdentificationErrorComponents`.
    """

    _pack_references = staticmethod(pack_references)
    _metric = "DiarizationErrorRate"

    def __init__(self, config: SpeakerDiarizationConfig, files: Iterable[Tuple[Optional[str], np.ndarray, Optional[Annotation]]],
                 sweep: Optional[HyperParameterSweep] = None, latencies: Optional[Iterable] = None,
                 uems: Optional[Sequence] = None, osp: Optional[Iterable[Mapping]] = None, speakers=None):
        self._sweep = sweep
        self.osp_sets = osp_sets(config, osp if osp is not None else ())
        self._speakers_arg = speakers
        super().__init__(config, files, latencies, uems)
        self.labels = [speaker_labels(k, config.max_speakers) for k in self.speakers]
        self._seeds = None
        if any(k is not None for k in self.speakers):
            # one seed table per clustering file: the files, or the latency units (each takes its file's centroids)
            if self.units is None:
                owner = list(range(len(self.uris)))
            else:
                owner = [0] * (len(self.units.unit_offsets) - 1)
                for li in range(len(self.latencies)):
                    for f in range(len(self.uris)):
                        owner[int(self.units.unit_of[li, f])] = f
            rows = [self.speakers[f].centroids if self.speakers[f] is not None else np.zeros((0, self.emb.shape[-1]))
                    for f in owner]
            self._seeds = (np.ascontiguousarray(np.cumsum([0] + [len(r) for r in rows]), dtype=np.int32),
                           np.ascontiguousarray(np.concatenate(rows), dtype=np.float64))

    def _check_speakers(self, chunk_samples: int):
        """``speakers`` -> ``self.speakers``, one KnownSpeakers or None per file (ValueError naming the file)"""
        speakers, nf, M = self._speakers_arg, len(self.uris), int(self.config.max_speakers)
        if speakers is None or isinstance(speakers, KnownSpeakers):
            speakers = [speakers] * nf
        elif not isinstance(speakers, (list, tuple)) or len(speakers) != nf:
            raise ValueError(f"speakers: need one KnownSpeakers for every file or one entry per file, {nf} in all")
        D = self._sweep.pipeline._native_models()[1].dims(chunk_samples)[1]
        out = []
        for f, known in enumerate(speakers):
            name = self.uris[f] if self.uris[f] is not None else f
            if known is not None and not isinstance(known, KnownSpeakers):
                raise ValueError(f"file {name}: speakers entry must be KnownSpeakers or None, not {type(known).__name__}")
            if known is not None and len(known) == 0:
                known = None
            if known is not None and known.dimension != D:
                raise ValueError(f"file {name}: the known speakers' centroids have dimension {known.dimension}, the "
                                 f"embeddings {D}")
            if known is not None and len(known) > M:
                raise ValueError(f"file {name}: {len(known)} known speakers, at most max_speakers = {M}")
            out.append(known)
        self.speakers: List[Optional[KnownSpeakers]] = out

    def _open(self) -> torch.device:
        if self._sweep is None:
            self._sweep = HyperParameterSweep(self.config)
        return self._sweep.device

    def _networks(self, fws: Sequence[FileWindows]):
        self._check_speakers(fws[0].chunk_samples)              # the models are open; nothing has run yet
        if len(self.osp_sets) == 1:
            self.seg, self.emb = self._sweep.network_pass_files(fws)
            self.embs = self.emb[None]
        else:
            self.seg, self.embs = self._sweep.network_pass_sets(fws, self.osp_sets)
            self.emb = self.embs[0]

    @property
    def resident_bytes(self) -> int:
        """device bytes of the kept network outputs"""
        return self.seg.numel() * self.seg.element_size() + self.embs.numel() * self.embs.element_size()

    def file_outputs(self, f: int, latency=None, osp: Optional[Mapping] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """file f's slice of the resident scores (n, F, K) and embeddings (n, K, D); ``latency`` (a constructed one, default
        the config's): its windows at that latency, the first chunks of its unit; ``osp`` (a constructed OSP set, keyed like
        the config; default the config's): that set's embeddings"""
        c0, c1 = self._chunk_range(f, latency)
        g = 0 if osp is None else osp_index(self.config, self.osp_sets, osp)
        return self.seg[c0:c1], self.embs[g, c0:c1]

    def _rows(self, trials: Sequence[Mapping[str, float]]) -> np.ndarray:
        """trials -> float64 (T, 4): :func:`trial_params` and the index of the trial's OSP set in :attr:`osp_sets`"""
        index, params = trial_osp_params(trials, self.config, self.osp_sets)
        return np.column_stack([params, index.astype(np.float64)])

    def _trial_sets(self, params: np.ndarray) -> Tuple[np.ndarray, torch.Tensor, Optional[Tuple[int, np.ndarray]]]:
        """params (T, 3), or (T, 4) with each trial's OSP set index -> (params (T, 3), the embeddings a launch reads, its
        trial sets): the resident embeddings of one set without trial sets when the sweep has one set or no set index is
        given, else those of all sets"""
        params = np.asarray(params, dtype=np.float64)
        if params.ndim == 2 and params.shape[1] == 4 and len(self.osp_sets) > 1:
            return params[:, :3], self.embs, (len(self.osp_sets), params[:, 3].astype(np.int32))
        return (params[:, :3] if params.ndim == 2 else params), self.emb, None

    def _over_files(self, entry, emb: torch.Tensor) -> tuple:
        """the leading arguments of ``HyperParameterSweep._run_trials`` / ``_score_trials`` for the ``_files`` entry point
        ``entry`` over the resident outputs and the concatenated plans"""
        nf = len(self.uris)
        return entry, (nf, self.offsets.ctypes.data), (nf,), self.seg, emb, (self.plan, self.out_start, self.out_res)

    def sweep(self, params: np.ndarray, keep_state: bool = False) -> SweepOutputs:
        """dg_sweep_run_files over the resident outputs for params (T, 3), or (T, 4) with each trial's OSP set index:
        header (T, N, 4) and turns over the N concatenated chunks; with ``keep_state`` maps (T, N, K) and centroids (files,
        T, M, D) on the device.  Not for a sweep built with ``latencies`` (:meth:`sweep_latencies`)."""
        if self.units is not None:
            raise ValueError("a sweep over several latencies runs through sweep_latencies")
        params, emb, sets = self._trial_sets(params)
        return self._sweep._run_trials(*self._over_files(_lib.lib().dg_sweep_run_files, emb), params, keep_state, sets,
                                       self._seeds)

    def run(self, trials: Sequence[Mapping[str, float]] = ({},)) -> List[List[Annotation]]:
        """-> predictions [file][trial]: what :meth:`HyperParameterSweep.run` returns for each file alone (with known
        speakers, what a pipeline seeded with the file's gives, its speakers labelled ``labels[f]``)"""
        if self.units is not None:
            return self.run_latencies(trials, [self.config.latency])[float(self.config.latency)]
        return self._run(self._rows(trials), self.sweep, self.labels)

    def score(self, trials: Sequence[Mapping[str, float]] = ({},), metric=None) \
            -> Tuple[List[DERComponents], DERComponents]:
        """-> (components per file, their sum in file order): per file what :meth:`HyperParameterSweep.score` returns for
        it alone with the same ``metric`` and the file's uem; ``total.der`` is the value ``Optimizer.objective``
        minimises.  Every file needs a reference.  With an :class:`IdentificationErrorRate` the components are
        :class:`IdentificationErrorComponents` (``total.ier``)."""
        if self.units is not None:
            return self.score_latencies(trials, [self.config.latency], metric)[float(self.config.latency)]
        return self._score(self._rows(trials), metric)

    def sweep_latencies(self, params: np.ndarray, latencies=None, keep_maps: bool = False) -> SweepOutputs:
        """dg_sweep_run_latencies over the resident outputs for params (T, 3) at the constructed ``latencies`` (None: all):
        header (T, Nv, 4), turns, out_start and out_res over the Nv virtual chunks (latency-major, then file order); with
        ``keep_maps`` the maps (T, N, K) over the N real chunks, on the device"""
        if self.units is None:
            raise ValueError("built without latencies: sweep_latencies needs DatasetSweep(..., latencies=...)")
        return self._sweep_virtual(params, self._tables(self._selection(latencies)), keep_maps)

    def run_latencies(self, trials: Sequence[Mapping[str, float]] = ({},), latencies=None) \
            -> Dict[float, List[List[Annotation]]]:
        """-> {latency: predictions [file][trial]} for the constructed ``latencies`` (None: all): for each latency L what
        :meth:`run` of a ``DatasetSweep`` built at L returns.  One launch per kernel and trial group for all of them."""
        params, sel = self._rows(trials), self._selection(latencies)
        if self.units is None:
            return {self.latencies[0]: self.run(trials)}
        return self._run_latencies(params, sel, self._sweep_virtual, self.labels)

    def score_latencies(self, trials: Sequence[Mapping[str, float]] = ({},), latencies=None, metric=None) \
            -> Dict[float, Tuple[List[DERComponents], DERComponents]]:
        """-> {latency: (components per file, their sum)} for the constructed ``latencies`` (None: all): for each latency L
        what :meth:`score` of a ``DatasetSweep`` built at L returns with the same ``metric``, bit for bit.  The clustering
        runs once per (unit, trial) whatever the number of latencies; one launch per kernel and trial group
        (:func:`trial_groups` over the virtual chunks)."""
        params, sel = self._rows(trials), self._selection(latencies)
        if self.units is None:
            return {self.latencies[0]: self.score(trials, metric)}
        return self._score_latencies(params, sel, self._score_virtual, metric)

    def _sweep_virtual(self, params: np.ndarray, tabs: tuple, keep_maps: bool = False) -> SweepOutputs:
        """one dg_sweep_run_latencies over the virtual layout ``tabs`` (``LatencyUnits.tables``)"""
        sw = self._sweep
        N, F, K = self.seg.shape
        h, _ = sw._handle(F, K, self.emb.shape[2], self.units.nw)
        params, emb, sets = self._trial_sets(params)
        _set_trial_sets(h, sets)
        _set_seeds(h, self._seeds)
        plan, out_start, out_res = tabs[2:5]
        params = np.ascontiguousarray(params, dtype=np.float64)
        T, Nv = len(params), len(tabs[0])
        header = np.empty((T, Nv, 4), dtype=np.int32)
        maps = torch.empty((T, N, K), dtype=torch.int32, device=self.device) if keep_maps else None
        n_turns, seconds = _turn_list_call(sw, self.device, T * Nv * 8, lambda *turn_list: _lib.lib().dg_sweep_run_latencies(
            h, self.seg.data_ptr(), emb.data_ptr(), *self._layout(tabs), params.ctypes.data, T, plan.ctypes.data,
            _lib.ptr(maps), header.ctypes.data, *turn_list))
        return SweepOutputs(header, sw._turns[:n_turns].copy(), n_turns, out_start, out_res, maps, None, seconds)

    def _score_virtual(self, params: np.ndarray, tabs: tuple, refs: tuple, regions: Optional[tuple]) \
            -> Tuple[np.ndarray, float]:
        """one dg_sweep_score_latencies over the virtual layout ``tabs`` against ``refs`` and ``regions`` (one entry per
        virtual file)"""
        N, F, K = self.seg.shape
        h, _ = self._sweep._handle(F, K, self.emb.shape[2], self.units.nw)
        _set_regions(_lib.lib().dg_sweep_set_scored_regions, h, regions)
        params, emb, sets = self._trial_sets(params)
        _set_trial_sets(h, sets)
        _set_seeds(h, self._seeds)
        _set_identities(h, refs[4] if len(refs) > 4 else None)
        plan, out_start, out_res, shifts = tabs[2:]
        params = np.ascontiguousarray(params, dtype=np.float64)
        comp = np.empty((len(tabs[1]) - 1, len(params), 5), dtype=np.float64)
        rc, seconds = _timed(self.device, lambda st: _lib.lib().dg_sweep_score_latencies(
            h, self.seg.data_ptr(), emb.data_ptr(), *self._layout(tabs), params.ctypes.data, len(params),
            plan.ctypes.data, out_start.ctypes.data, out_res.ctypes.data, shifts.ctypes.data, PATCH_COLLAR,
            *(a.ctypes.data for a in refs[:4]), comp.ctypes.data, st))
        _lib.check(rc)
        return comp, seconds()

    def _score_group(self, params: np.ndarray, refs: tuple, regions: Optional[tuple]) -> Tuple[np.ndarray, float]:
        reference = tuple(a.ctypes.data for a in refs[:4])         # rows, labels, row offsets, label counts
        params, emb, sets = self._trial_sets(params)
        return self._sweep._score_trials(*self._over_files(_lib.lib().dg_sweep_score_files, emb), params,
                                         self.shifts.ctypes.data, reference, regions=regions, trial_sets=sets,
                                         seeds=self._seeds, identities=refs[4] if len(refs) > 4 else None)[:2]

    def _metric_kind(self, metric) -> Tuple[str, float, bool]:
        return diarization_metric(metric)

    def _pack(self, kind: str, references: List[Annotation], regions: Optional[list], copies: int) -> tuple:
        """``pack_references``; for the identification error rate followed by the name table (:func:`pack_identities`)"""
        refs = pack_references(references, regions)
        if kind == "IdentificationErrorRate":
            refs = (*refs, pack_identities(references, regions, self.labels * copies))
        return refs

    def _components(self, f: int, comp: np.ndarray, refs: tuple) -> DERComponents:
        return (IdentificationErrorComponents if len(refs) > 4 else DERComponents).from_array(comp)


VAD_PARAMS = tuple(hp.name for hp in VoiceActivityDetection.hyper_parameters())   # ("tau_active",)


@dataclass
class DetectionErrorComponents:
    """Detection error rate components in seconds, one entry per trial (float64 (T,) each)."""
    false_alarm: np.ndarray
    missed_detection: np.ndarray
    total: np.ndarray

    def as_array(self) -> np.ndarray:
        """(T, 3) {false alarm, missed detection, total}"""
        return np.stack([self.false_alarm, self.missed_detection, self.total], axis=1)

    @property
    def detection_error_rate(self) -> np.ndarray:
        """(false alarm + missed detection) / total per trial (:func:`_rate`)"""
        return _rate(self.false_alarm + self.missed_detection, self.total)

    def __add__(self, other: "DetectionErrorComponents") -> "DetectionErrorComponents":
        """the components of several files summed per trial"""
        return DetectionErrorComponents(self.false_alarm + other.false_alarm,
                                        self.missed_detection + other.missed_detection, self.total + other.total)


def speech_reference(annotation: Annotation, regions: Optional[Sequence[Tuple[float, float]]] = None) \
        -> Tuple[np.ndarray, float]:
    """A reference annotation -> (rows float64 (S, 2), total): the support of all its segments, whatever their labels
    (``annotation.get_timeline().support()``): non-empty segments in (start, end) order, a segment merged into the current
    row when ``Segment(row end, its start)`` is falsy (it overlaps, touches or follows by at most 1e-6 s).  ``total`` is the
    rows' durations summed in order, pyannote's ``reference.duration()``.  With ``regions`` (:func:`scored_regions`) the
    segments are first cropped to them (:func:`cropped_tracks`), so ``total`` is the cropped support's duration."""
    rows: List[List[float]] = []
    for a, b in sorted((s, e) for s, e, _ in cropped_tracks(annotation, regions)):
        if rows and not (a - rows[-1][1] > 1e-6):
            rows[-1][1] = max(rows[-1][1], b)
        else:
            rows.append([a, b])
    total = 0.0
    for a, b in rows:
        total += b - a
    return np.array(rows, dtype=np.float64).reshape(-1, 2), total


def pack_speech_references(references: Sequence[Annotation], regions: Optional[Sequence] = None):
    """per-file references -> the reference arguments of dg_vad_sweep_score_files and the per-file totals: (rows float64
    (S, 2), row offsets int32 (files + 1,), totals float64 (files,)), cropped to each file's entry of ``regions`` when given"""
    rows, offsets, totals = [], [0], []
    for f, ref in enumerate(references):
        r, total = speech_reference(ref, None if regions is None else regions[f])
        rows.append(r)
        offsets.append(offsets[-1] + len(r))
        totals.append(total)
    return (np.ascontiguousarray(np.concatenate(rows), dtype=np.float64), np.array(offsets, dtype=np.int32),
            np.array(totals, dtype=np.float64))


class VoiceActivitySweep(_DatasetSweep):
    """Tunes ``VoiceActivityDetection``'s ``tau_active`` over a whole dataset with the segmentation run once.

        vs = VoiceActivitySweep(vad_config, [("file1", waveform1, reference1), ("file2", waveform2, reference2)])
        per_file, total = vs.score([{"tau_active": 0.4}, {"tau_active": 0.55}, {}])
        best = int(np.argmin(total.detection_error_rate))

    ``files``: (uri, 1-D float32 waveform at ``config.sample_rate``, reference annotation or None).  The constructor runs the
    segmentation of every file's windows (``DeviceAudioStream`` batches of 256 from the file's window 0, the
    ``SpeakerSegmentation.forward_device`` call ``VoiceActivityDetection`` makes) as one flow without synchronising, keeps
    the scores on the device (F K float32 per chunk: 3.5 kB at the default model) and computes the speech curve once
    (``dg_vad_sweep_curve``: max over the local speakers, Hamming aggregation; 29 float64 per chunk at the defaults).
    :meth:`score` and :meth:`run` then threshold the curve for every (file, trial) pair in one launch per kernel and per
    trial group (:func:`trial_groups`), and run no network kernel.  The windows, plans and timestamp shifts are those of
    :class:`DatasetSweep`.  Needs the native segmentation model (``B200PyanNet``).  ``uems`` and the ``metric`` of
    :meth:`score` / :meth:`score_latencies` (a :class:`DetectionErrorRate`, or pyannote.metrics' own) as in
    :class:`DatasetSweep`.
    """

    _pack_references = staticmethod(pack_speech_references)
    _stream_form = False      # forward_device passes no hop hint: the per-window form for every batch
    _metric = "DetectionErrorRate"

    def __init__(self, config: VoiceActivityDetectionConfig,
                 files: Iterable[Tuple[Optional[str], np.ndarray, Optional[Annotation]]], latencies: Optional[Iterable] = None,
                 uems: Optional[Sequence] = None):
        self._h: Optional[C.c_void_p] = None
        self._turns = np.empty(0, dtype=np.uint32)
        super().__init__(config, files, latencies, uems)
        t1 = time.perf_counter()
        N, F, K = self.seg.shape
        if self.units is None:
            plan, nw = self.plan, int(round(config.latency / config.step))
        else:                              # the curve of every (latency, file) pair, over the virtual chunks
            plan, nw = self._tables(range(len(self.latencies)))[2], self.units.nw
        self.curve_frames = int(np.where(plan[:, 2] > 0, plan[:, 2], plan[:, 1]).sum())
        ham = np.ascontiguousarray(np.hamming(F), dtype=np.float64)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_vad_sweep_create(F, K, nw, ham.ctypes.data, self.device.index, C.byref(h)))
            self._h = h
            if self.units is None:
                _lib.check(_lib.lib().dg_vad_sweep_curve(h, self.seg.data_ptr(), N, len(self.uris), self.offsets.ctypes.data,
                                                         self.plan.ctypes.data, _lib.stream_ptr(self.device)))
            else:
                tabs = self._tables(range(len(self.latencies)))
                _lib.check(_lib.lib().dg_vad_sweep_curve_latencies(h, self.seg.data_ptr(), *self._layout(tabs),
                                                                   tabs[2].ctypes.data, _lib.stream_ptr(self.device)))
        self.timing["curve"] = time.perf_counter() - t1

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                _lib.lib().dg_vad_sweep_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    def _open(self) -> torch.device:
        self.pipeline = VoiceActivityDetection(self.config)
        if not isinstance(getattr(self.pipeline.segmentation.model, "model", None), B200PyanNet):
            raise _lib.DiartB200Error("VoiceActivitySweep needs the native segmentation model (B200PyanNet)")
        return _indexed(self.pipeline.segmentation.device)

    def _networks(self, fws: Sequence[FileWindows]):
        """scores (N, F, K) of every window of every file, concatenated in file order, on the device: each file's windows in
        batches cut at the multiples of 256 from its window 0, so that a file's scores are the bits
        ``VoiceActivityDetection`` computes for it in batches of 256"""
        seg = self.pipeline.segmentation
        batches = FileBatches(fws, self.config, self.device)
        with torch.cuda.device(self.device):
            self.seg = torch.cat([seg.forward_device(windows) for windows in batches])

    @property
    def resident_bytes(self) -> int:
        """device bytes of the kept scores and speech curve"""
        return self.seg.numel() * self.seg.element_size() + self.curve_frames * 8

    def file_outputs(self, f: int, latency=None) -> torch.Tensor:
        """file f's slice of the resident scores (n, F, K); ``latency`` (a constructed one, default the config's): its windows
        at that latency, the first chunks of its unit"""
        c0, c1 = self._chunk_range(f, latency)
        return self.seg[c0:c1]

    def _taus(self, trials: Sequence[Mapping[str, float]]) -> np.ndarray:
        return np.ascontiguousarray(trial_params(trials, self.config, VAD_PARAMS)[:, 0])

    def binarize(self, taus: np.ndarray) -> SweepOutputs:
        """dg_vad_sweep_run_files for thresholds (T,): header (T, N, 4) and turns over the N concatenated chunks (for a
        sweep built with ``latencies``, the virtual chunks of every latency)"""
        taus = np.ascontiguousarray(taus, dtype=np.float64)
        T, N = len(taus), self.num_chunks if self.units is None else len(self._tables(self._launched([]))[0])
        header = np.empty((T, N, 4), dtype=np.int32)
        n_turns, seconds = _turn_list_call(self, self.device, T * N * 4, lambda *turn_list: _lib.lib().dg_vad_sweep_run_files(
            self._h, taus.ctypes.data, T, header.ctypes.data, *turn_list))
        out_start, out_res = (self.out_start, self.out_res) if self.units is None else self._tables(self._launched([]))[3:5]
        return SweepOutputs(header, self._turns[:n_turns].copy(), n_turns, out_start, out_res, device_seconds=seconds)

    def run(self, trials: Sequence[Mapping[str, float]] = ({},)) -> List[List[Annotation]]:
        """-> predictions [file][trial]: for each file and trial what ``Benchmark.run_single`` returns for
        ``VoiceActivityDetection`` with that tau_active (label "speech", modality "speech", the file's uri)"""
        if self.units is not None:
            return self.run_latencies(trials, [self.config.latency])[float(self.config.latency)]
        out = self._run(self._taus(trials), self.binarize, [["speech"]] * len(self.uris))
        for preds in out:
            for p in preds:                # the per-chunk VAD annotations carry modality "speech" whatever the shift
                p.modality = "speech"
        return out

    def score(self, trials: Sequence[Mapping[str, float]] = ({},), metric=None) \
            -> Tuple[List[DetectionErrorComponents], DetectionErrorComponents]:
        """-> (components per file, their sum in file order): the detection error rate components of :meth:`run`'s
        predictions against each file's reference under ``metric`` (default ``DetectionErrorRate(collar=0,
        skip_overlap=False)``) within the file's uem (default: none); the minimum of ``total.detection_error_rate`` is the
        trial ``Optimizer.objective`` would pick.  Every file needs a reference."""
        if self.units is not None:
            return self.score_latencies(trials, [self.config.latency], metric)[float(self.config.latency)]
        return self._score(self._taus(trials), metric)

    def run_latencies(self, trials: Sequence[Mapping[str, float]] = ({},), latencies=None) \
            -> Dict[float, List[List[Annotation]]]:
        """-> {latency: predictions [file][trial]} for the constructed ``latencies`` (None: all): for each latency L what
        :meth:`run` of a ``VoiceActivitySweep`` built at L returns.  The thresholds run over the curve of every constructed
        latency (computed once, by the constructor), one launch per kernel and trial group."""
        taus, sel = self._taus(trials), self._selection(latencies)
        if self.units is None:
            return {self.latencies[0]: self.run(trials)}
        out = self._run_latencies(taus, sel, lambda t, tabs: self.binarize(t), [["speech"]] * len(self.uris))
        for runs in out.values():
            for preds in runs:
                for p in preds:
                    p.modality = "speech"
        return out

    def score_latencies(self, trials: Sequence[Mapping[str, float]] = ({},), latencies=None, metric=None) \
            -> Dict[float, Tuple[List[DetectionErrorComponents], DetectionErrorComponents]]:
        """-> {latency: (components per file, their sum)} for the constructed ``latencies`` (None: all): for each latency L
        what :meth:`score` of a ``VoiceActivitySweep`` built at L returns with the same ``metric``, bit for bit.  One launch
        per kernel and trial group over every constructed latency."""
        taus, sel = self._taus(trials), self._selection(latencies)
        if self.units is None:
            return {self.latencies[0]: self.score(trials, metric)}
        return self._score_latencies(taus, sel, lambda t, tabs, refs, regions: self._vad_score(t, *tabs[3:6], refs, regions),
                                     metric)

    def _launched(self, sel: List[int]) -> List[int]:
        return list(range(len(self.latencies)))       # the curve covers every constructed latency

    def _group_chunks(self, tabs: tuple) -> int:
        return len(tabs[0])                            # no clustering: header and turns over the virtual chunks

    def _score_group(self, taus: np.ndarray, refs: tuple, regions: Optional[tuple]) -> Tuple[np.ndarray, float]:
        return self._vad_score(taus, self.out_start, self.out_res, self.shifts, refs, regions)

    def _vad_score(self, taus: np.ndarray, out_start: np.ndarray, out_res: np.ndarray, shifts: np.ndarray,
                   refs: tuple, regions: Optional[tuple] = None) -> Tuple[np.ndarray, float]:
        """one dg_vad_sweep_score_files against ``refs`` (``pack_speech_references`` of the curve's files), the hypotheses
        cropped to ``regions`` (or None) -> (components (files, T, 2), device seconds)"""
        rows, roff, _ = refs
        taus = np.ascontiguousarray(taus)
        _set_regions(_lib.lib().dg_vad_sweep_set_scored_regions, self._h, regions)
        part = np.empty((len(roff) - 1, len(taus), 2), dtype=np.float64)
        rc, seconds = _timed(self.device, lambda st: _lib.lib().dg_vad_sweep_score_files(
            self._h, taus.ctypes.data, len(taus), out_start.ctypes.data, out_res.ctypes.data,
            shifts.ctypes.data, PATCH_COLLAR, rows.ctypes.data, roff.ctypes.data, part.ctypes.data, st))
        _lib.check(rc)
        return part, seconds()

    def _components(self, f: int, comp: np.ndarray, refs: tuple) -> DetectionErrorComponents:
        """false alarm and missed detection from the device; the total is the (cropped) reference's duration, whatever the
        trial"""
        return DetectionErrorComponents(comp[:, 0].copy(), comp[:, 1].copy(), np.full(len(comp), refs[2][f]))
