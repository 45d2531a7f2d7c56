"""Many live audio streams on one GPU (``dg_multi``, ``csrc/api_multi.cu``).

The reference serves a live stream with ``StreamingInference(batch_size=1)``: one 5 s window every 0.5 s, each a separate
``SpeakerDiarization.__call__`` (``diart.stream`` / ``diart.serve``).  N streams on one GPU would be N batch-1 network passes
per step.  ``MultiStreamDiarization`` owns up to ``max_streams`` streams with one configuration and the same native models and
serves them in ticks: every open stream gives its complete, unconsumed windows (at most ``max_windows_per_stream``), and all
of them run as one batch -- one upload of the new audio, one network pass, one clustering launch with a state per stream,
one post-path launch with an aggregation history per stream.  A stream's scores are bit-identical to those its own
``SpeakerDiarization`` computes on its windows one at a time, and so are the post-path's arithmetic and plan.  Its
embeddings can differ in the last bits (the fused TDNN5 pooling groups its partial sums by a window's row in the batch), so
a clustering decision that lies exactly at a threshold could go the other way; apart from that the speaker maps and turns
are the dedicated pipeline's.  Only the turns come back (the reference's serve hook writes RTTM, no audio).

Streams at other source rates (``source_sample_rates``; ``open(sample_rate=44100)``) are windowed at their own rate, as
``rearrange_audio_stream(duration, step, rate)`` windows them, and every window is resampled on the device with the bits of
``DeviceResample`` on that window (the reference's ``blocks.Resample``): each 16 kHz frame inside the windows is computed once
per stream, only the frames at each window's edges once per window.

``MultiStreamVoiceActivityDetection`` serves the reference's ``VoiceActivityDetection`` the same way (``dg_multi_create_vad``):
the same audio path, the segmentation network alone, and every stream's speech curve aggregated and binarised on the device.
Its results carry no caveat: they are bit for bit those of a dedicated ``VoiceActivityDetection``.

Each stream may have its own latency (up to the server's ``max_latency``) and thresholds (``open(latency=...,
tau_active=...)``, and ``rho_update`` / ``delta_new`` for diarization), none of which reaches the networks: the tick's one
network pass is shared, the clustering runs every stream's state at that stream's thresholds, and the post-path aggregates
each stream's own number of buffers and binarises at its own ``tau_active``.  A stream's results are then those of a
dedicated pipeline whose configuration is the server's with that stream's values.

A diarization stream may also start from known speakers (``open(speakers=...)``, ``diart_b200.speakers``): its clustering
state is seeded with their centroids and its annotations name them; ``speakers(sid)`` exports a stream's state, so that a
closed stream can be resumed with the same centroids and labels.  With a ``gallery`` (``speakers.SpeakerGallery``), every tick
also names the streams' discovered speakers from it on the device; ``open(gallery=...)`` gives a stream its own gallery and
threshold instead, and one grouped search per tick serves every gallery in use.

``export(sids)`` takes streams out of a server with their whole state (``transfer.StreamState``), and ``restore(states)``
opens them in this or another compatible server, on this or another GPU or machine: the next tick continues each stream
bit for bit as if it had never moved.  ``export(sids, close=False)`` is a checkpoint that leaves the streams running."""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _lib
from . import models as m
from .blocks.diarization import SpeakerDiarizationConfig
from .blocks.post import chunk_annotations, crop_plan, turn_capacity
from .blocks.vad import VoiceActivityDetectionConfig, speech_annotations
from .core import Annotation
from .operators import DeviceResample
from .speakers import KnownSpeakers, SpeakerGallery, check_gallery, exported, speaker_labels
from .transfer import VERSION as STATE_VERSION
from .transfer import StreamState, gallery_fingerprint, model_fingerprint


def plan_rows(idx: np.ndarray, step: float, window_samples: int, sample_rate: int, frames: int, nw: int, latency: float,
              resolution=None):
    """The post-path plan rows (``blocks.post.post_plan``) of chunks ``idx`` (B,) of streams whose window i starts at
    ``i * step`` and is fed to its pipeline one window per call -> (plan int32 (B, 4 + nw), out_start (B,), out_res (B,)).
    A row depends only on the chunk's index within its stream, so one vectorised evaluation covers every stream of a tick.
    Each buffer has its own start time and score resolution (extent duration / frames of its window, as
    ``SpeakerDiarization.__call__`` measures it).  ``resolution``: the sample spacing of each row's window, scalar or (B,)
    (default ``1 / sample_rate``; a resampled stream's is ``(chunk / source rate) / window_samples``)."""
    idx = np.asarray(idx, dtype=np.int64)
    res_row = 1 / sample_rate if resolution is None else np.asarray(resolution, dtype=np.float64)
    win = np.broadcast_to(window_samples * res_row, idx.shape)   # SlidingWindowFeature.extent: start + n * step

    def start_res(k, w):
        s = k * step
        e = s + w
        return s, np.where(e > s, e - s, 0.0) / frames       # Segment.duration / frames

    starts, res = start_res(idx.astype(np.float64), win)
    nb = np.minimum(idx + 1, nw)
    j = np.arange(nw)[None, :]
    valid = j < nb[:, None]
    s_j, r_j = start_res(np.where(valid, (idx - (nb - 1))[:, None] + j, 0).astype(np.float64), win[:, None])
    return crop_plan(starts, res, s_j, r_j, nb, valid, nw, frames, step, latency)


def same_device(a, b) -> bool:
    """whether torch devices ``a`` and ``b`` are the same CUDA device (an index-less ``cuda`` is the current one)"""
    a, b = torch.device(a), torch.device(b)
    if a.type != b.type:
        return False
    if a.type != "cuda":
        return True
    index = lambda d: d.index if d.index is not None else torch.cuda.current_device()  # noqa: E731
    return index(a) == index(b)


def available_windows(pushed: np.ndarray, emitted: np.ndarray, window_samples, step_samples) -> np.ndarray:
    """complete windows of streams that received ``pushed`` samples and gave ``emitted`` windows (dg_multi_available);
    window and step samples are scalars or per stream"""
    have = pushed - emitted * step_samples
    return np.where(have >= window_samples, (have - window_samples) // np.maximum(step_samples, 1) + 1, 0)


def source_geometry(rate: int, sample_rate: int, duration: float, step: float) -> Tuple[int, int, float]:
    """(chunk, step samples, window resolution) of a stream at source ``rate`` served by a pipeline at ``sample_rate``, as
    ``DeviceAudioStream(source_sample_rate=rate)`` windows and time-stamps it.  ValueError unless the chunk resamples to the
    pipeline's chunk and a step is a whole number of resampled frames (``step % o == 0``, ``o / n`` the reduced ratio)."""
    rate, sample_rate = int(rate), int(sample_rate)
    if rate < 1:
        raise ValueError(f"sample rate {rate} must be positive")
    chunk, hop = int(round(rate * duration)), int(round(rate * step))
    window = int(np.rint(duration * sample_rate))
    if rate == sample_rate:
        return chunk, hop, 1 / sample_rate
    o = rate // math.gcd(rate, sample_rate)
    n = sample_rate // math.gcd(rate, sample_rate)
    out = -(-n * chunk // o)
    if out != window:
        raise ValueError(f"a {duration} s chunk at {rate} Hz ({chunk} samples) resamples to {out} samples, not the "
                         f"pipeline's {window}")
    if hop < 1 or hop % o:
        raise ValueError(f"a {step} s step at {rate} Hz ({hop} samples) is not a whole number of resampled frames "
                         f"({o} source samples each)")
    return chunk, hop, (chunk * (1 / rate)) / window


def stream_windows(latency: float, step: float) -> int:
    """the buffers a stream at ``latency`` aggregates (``DelayedAggregation.num_overlapping_windows``)"""
    return int(round(latency / step))


def mixed_plan(idx: np.ndarray, latency: np.ndarray, step: float, window_samples: int, sample_rate: int, frames: int,
               nw: int, resolution):
    """``plan_rows`` of a tick whose rows (chunk indices ``idx`` (B,), row latencies ``latency`` (B,), window resolutions
    ``resolution`` (B,)) belong to streams at several latencies: one ``plan_rows`` per distinct latency, its rows scattered
    into plan int32 (B, 4 + nw), ``nw`` the largest number of buffers of any stream; a row with fewer buffers leaves the tail
    0.  -> (plan, out_start (B,), out_res (B,))"""
    idx = np.asarray(idx, dtype=np.int64)
    latency = np.asarray(latency, dtype=np.float64)
    res = np.broadcast_to(np.asarray(resolution, dtype=np.float64), idx.shape)
    lats = np.unique(latency)
    if len(lats) <= 1 and (len(lats) == 0 or stream_windows(lats[0], step) == nw):   # one latency: one evaluation
        lat = float(lats[0]) if len(lats) else step * nw
        return plan_rows(idx, step, window_samples, sample_rate, frames, nw, lat, res)
    plan = np.zeros((len(idx), 4 + nw), dtype=np.int32)
    out_start, out_res = np.empty(len(idx)), np.empty(len(idx))
    for lat in lats.tolist():
        rows = np.flatnonzero(latency == lat)
        p, s, r = plan_rows(idx[rows], step, window_samples, sample_rate, frames, stream_windows(lat, step), lat, res[rows])
        plan[rows, :p.shape[1]] = p
        out_start[rows], out_res[rows] = s, r
    return plan, out_start, out_res


class _MultiStreamServer:
    """What the multi-stream servers share: the ``dg_multi`` handle a subclass creates (``_create``), the declared source
    rates, the host mirror of the slots (``open`` / ``close`` / ``push`` / ``available``) and the planning of a tick."""

    _needs = ""   # what the subclass raises when a model is not native

    def __init__(self, config, max_streams: int, max_windows_per_stream: int, source_sample_rates, models, max_latency=None):
        self._h: Optional[C.c_void_p] = None
        self.config = config
        msg = f"Latency should be in the range [{config.step}, {config.duration}]"
        assert config.step <= config.latency <= config.duration, msg
        self.max_latency = float(config.latency if max_latency is None else max_latency)
        if not config.latency <= self.max_latency <= config.duration:
            raise ValueError(f"max_latency {self.max_latency} should be in the range [{config.latency}, {config.duration}] "
                             "(the configuration's latency, its duration)")
        for lazy in models:
            lazy.eval()
            lazy.to(config.device)
        seg_net = config.segmentation.model
        if not isinstance(seg_net, m.B200PyanNet):
            raise _lib.DiartB200Error(self._needs)
        sr = config.sample_rate
        self.window_samples = int(np.rint(config.duration * sr))
        self.step_samples = int(round(config.step * sr))
        self.max_streams, self.max_windows_per_stream = int(max_streams), int(max_windows_per_stream)
        self.F, self.K = seg_net.dims(self.window_samples)
        self.nw = stream_windows(self.max_latency, config.step)   # the most buffers a stream aggregates (plan width - 4)
        self.device = seg_net.device
        ham = np.ascontiguousarray(np.hamming(self.F), dtype=np.float64)
        self._h = self._create(ham)
        # rate -> (rate id, chunk samples, step samples, window resolution); one DeviceResample (tap table) per declared rate
        self.rates = {sr: (-1, self.window_samples, self.step_samples, 1 / sr)}
        self._resamplers: Dict[int, DeviceResample] = {}
        for rate in sorted({int(r) for r in source_sample_rates} - {sr}):
            chunk, hop, res = source_geometry(rate, sr, config.duration, config.step)
            rs = DeviceResample(rate, sr, self.device)
            rid = C.c_int()
            with torch.cuda.device(self.device):
                _lib.check(_lib.lib().dg_multi_add_rate(self._h, rs.handle, chunk, hop, C.byref(rid)))
            self._resamplers[rate] = rs
            self.rates[rate] = (rid.value, chunk, hop, res)
        # host mirror of the slots: open, samples pushed, windows consumed, timestamp shift, window / step samples and
        # resolution at the stream's rate
        self._open = np.zeros(self.max_streams, dtype=bool)
        self._pushed = np.zeros(self.max_streams, dtype=np.int64)
        self._emitted = np.zeros(self.max_streams, dtype=np.int64)
        self._shift = np.zeros(self.max_streams, dtype=np.float64)
        self._chunk = np.full(self.max_streams, self.window_samples, dtype=np.int64)
        self._hop = np.full(self.max_streams, self.step_samples, dtype=np.int64)
        self._res = np.full(self.max_streams, 1 / sr, dtype=np.float64)
        self._latency = np.full(self.max_streams, float(config.latency), dtype=np.float64)   # each stream's latency
        self._turns = np.empty(1 << 16, dtype=np.uint32)

    def _create(self, hamming: np.ndarray) -> C.c_void_p:
        """the handle (dg_multi_create*)"""
        raise NotImplementedError

    def _outputs(self, B: int) -> tuple:
        """the device tensors a tick with ``outputs`` fills: (scores, embeddings, maps), None where the handle has none"""
        raise NotImplementedError

    def _annotations(self, header, turns, n_turns, out_start, out_res, shifts) -> List[Annotation]:
        """the tick's annotations; ``shifts``: the timestamp shift of each row (``_row_sids``: its stream)"""
        raise NotImplementedError

    def _after_tick(self, B: int):
        """called once a tick of B windows has run, before its annotations are built"""

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                _lib.lib().dg_multi_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def _open_stream(self, shift: float, sample_rate: Optional[int], latency: Optional[float],
                     seed: Optional[np.ndarray] = None, **thresholds) -> int:
        """a new stream (fresh clustering and aggregation state) in the lowest free slot, its blocks at ``sample_rate``
        (default: the pipeline's; otherwise one of ``source_sample_rates``), at its own ``latency`` and ``thresholds``
        (name -> value, in the order of the handle's {tau, rho, delta}; None: the config's).  ``seed``: known centroids
        float64 (n, D) its clustering state starts from (dg_multi_open_seeded).  Everything is checked before the handle is
        touched: a refusal raises ValueError and leaves the slot closed.  Returns the stream's id"""
        cfg = self.config
        rate = cfg.sample_rate if sample_rate is None else int(sample_rate)
        if rate not in self.rates:
            raise ValueError(f"sample rate {rate} was not declared (source_sample_rates: {sorted(self._resamplers)})")
        lat = float(cfg.latency if latency is None else latency)
        if not cfg.step <= lat <= self.max_latency:
            raise ValueError(f"latency {lat} should be in the range [{cfg.step}, {self.max_latency}] (step, max_latency)")
        params = np.zeros(3, dtype=np.float64)
        for i, (name, value) in enumerate(thresholds.items()):
            params[i] = float(getattr(cfg, name) if value is None else value)
            if not math.isfinite(params[i]):
                raise ValueError(f"{name} must be finite, not {params[i]}")
        free = np.flatnonzero(~self._open)
        if len(free) == 0:
            raise ValueError(f"all {self.max_streams} streams are open")
        sid = int(free[0])
        rid = self.rates[rate][0]
        with torch.cuda.device(self.device):
            if seed is None:
                _lib.check(_lib.lib().dg_multi_open_config(self._h, sid, rid, stream_windows(lat, cfg.step),
                                                           params.ctypes.data))
            else:
                seed = np.ascontiguousarray(seed, dtype=np.float64)
                _lib.check(_lib.lib().dg_multi_open_seeded(self._h, sid, rid, stream_windows(lat, cfg.step),
                                                           params.ctypes.data, seed.ctypes.data, len(seed)))
        self._begin(sid, rate, lat, shift, 0, 0)
        return sid

    def _begin(self, sid: int, rate: int, latency: float, shift: float, pushed: int, emitted: int):
        """the host mirror of a stream that starts in slot ``sid`` (new or restored): at source ``rate`` and ``latency``,
        time stamps shifted by ``shift``, ``pushed`` samples pushed and ``emitted`` windows consumed so far"""
        self._open[sid] = True
        self._pushed[sid], self._emitted[sid] = pushed, emitted
        self._shift[sid] = float(shift)
        _, self._chunk[sid], self._hop[sid], self._res[sid] = self.rates[rate]
        self._latency[sid] = latency

    def close(self, sid: int):
        _lib.check(_lib.lib().dg_multi_close(self._h, int(sid)))
        self._release(sid)

    def _release(self, sid: int):
        """the host mirror of a slot that was closed"""
        self._open[sid] = False

    _kind = ""   # StreamState.kind of the subclass's streams

    def _settings(self) -> dict:
        """what a stream's results depend on besides its own values and the models: a restored state must have them"""
        cfg = self.config
        return dict(duration=float(cfg.duration), step=float(cfg.step), sample_rate=int(cfg.sample_rate),
                    window_samples=self.window_samples, step_samples=self.step_samples, F=self.F, K=self.K)

    def _models(self) -> list:
        return [model_fingerprint(self.config.segmentation.model)]

    def _stream_meta(self, sid: int) -> dict:
        """the host part of stream ``sid``'s state"""
        rate = next(r for r, (rid, chunk, hop, res) in self.rates.items() if chunk == self._chunk[sid] and
                    hop == self._hop[sid] and res == self._res[sid])
        return dict(version=STATE_VERSION, kind=self._kind, models=self._models(), settings=self._settings(), rate=rate,
                    latency=float(self._latency[sid]), shift=float(self._shift[sid]), pushed=int(self._pushed[sid]),
                    emitted=int(self._emitted[sid]))

    def _restore_gallery(self, state: StreamState, gallery):
        """the gallery state ``state`` is named from here (None: none), or ValueError"""
        return None

    def _restored(self, sid: int, state: StreamState, gallery):
        """the host mirror of a slot a state was restored into"""
        meta = state._meta
        self._begin(sid, meta["rate"], meta["latency"], meta["shift"], meta["pushed"], meta["emitted"])

    def export(self, sids, *, close: bool = True) -> List[StreamState]:
        """the whole state of each open stream in ``sids`` after the last tick, its samples pushed since then included, in
        one launch and one copy (per 256 MiB).  ``close=True`` closes the streams as ``close`` does; ``close=False`` leaves
        them running untouched (a checkpoint).  ValueError, closing nothing, for a stream that is not open or listed twice;
        AssertionError for a diarization stream in the "Cannot update unknown centers" state (as ``speakers``)."""
        sids = [int(s) for s in sids]
        for s in sids:
            if not (0 <= s < self.max_streams and self._open[s]):
                raise ValueError(f"stream {s} is not open")
        slots = np.asarray(sids, dtype=np.int32)
        sizes = np.zeros(len(sids), dtype=np.int64)
        lib = _lib.lib()
        _lib.check(lib.dg_multi_export_bytes(self._h, slots.ctypes.data, len(sids), sizes.ctypes.data))
        out = np.empty(int(sizes.sum()), dtype=np.uint8)
        with torch.cuda.device(self.device):
            _lib.check(lib.dg_multi_export(self._h, slots.ctypes.data, len(sids), int(bool(close)), out.ctypes.data,
                                           len(out)))
        off = np.concatenate([[0], np.cumsum(sizes)])
        # each state views its part of the one output buffer (no second copy of a drain's gigabytes)
        states = [StreamState(out[off[a]:off[a + 1]], self._stream_meta(s)) for a, s in enumerate(sids)]
        if close:
            for s in sids:
                self._release(s)
        return states

    def restore(self, states, *, gallery=None) -> List[int]:
        """opens each exported state in the lowest free slot, in order, with everything it had (counters, timestamp
        shift, source rate, latency, thresholds, history, clustering, labels, names and claims): the next ``step``
        continues each stream as if it had never left.  ``gallery``: the gallery of the states named from one (one
        ``SpeakerGallery`` for all, or one entry per state; None: the server's default); it must be the very gallery the
        stream was named from (same names and centroids), and the stream keeps its own threshold.  Returns the stream ids.
        ValueError, naming the reason, with every slot left closed and nothing launched: another kind of stream, other
        models or settings, a latency above ``max_latency``, an undeclared source rate, a backlog beyond the ring, a
        missing or different gallery, no free slot, another format version."""
        states = list(states)
        n = len(states)
        gals = list(gallery) if isinstance(gallery, (list, tuple)) else [gallery] * n
        if len(gals) != n:
            raise ValueError(f"{len(gals)} galleries for {n} states")
        models, settings = self._models(), self._settings()
        use = []
        for a, st in enumerate(states):
            if not isinstance(st, StreamState):
                raise TypeError(f"states[{a}]: expected StreamState, got {type(st).__name__}")
            meta = st._meta
            if meta.get("version") != STATE_VERSION:
                raise ValueError(f"state {a} has format version {meta.get('version')}; this build reads {STATE_VERSION}")
            if meta["kind"] != self._kind:
                raise ValueError(f"state {a} is a {meta['kind']} stream, this server serves {self._kind} streams")
            if meta["models"] != models:
                raise ValueError(f"state {a} was computed with other models")
            if meta["settings"] != settings:
                diff = sorted(k for k in settings if meta["settings"].get(k) != settings[k])
                raise ValueError(f"state {a} was computed with other settings: {', '.join(diff)}")
            if not meta["latency"] <= self.max_latency:
                raise ValueError(f"state {a} has latency {meta['latency']}, above this server's max_latency "
                                 f"{self.max_latency}")
            if meta["rate"] not in self.rates:
                raise ValueError(f"state {a} is at {meta['rate']} Hz, a rate this server did not declare "
                                 f"(source_sample_rates: {sorted(self._resamplers)})")
            use.append(self._restore_gallery(st, gals[a]))
        if n > int((~self._open).sum()):
            raise ValueError(f"{n} states, {int((~self._open).sum())} free slots")
        blob = np.concatenate([st._blob for st in states]) if n else np.empty(0, np.uint8)
        handles = (C.c_void_p * max(n, 1))(*[None if g is None else g.handle for g in use])
        slots = np.empty(max(n, 1), dtype=np.int32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_multi_import(self._h, blob.ctypes.data, len(blob), n, handles, slots.ctypes.data))
        sids = slots[:n].tolist()
        for sid, st, g in zip(sids, states, use):
            self._restored(sid, st, g)
        return sids

    def push(self, sid: int, block: np.ndarray):
        """appends a block of samples, shape (n,), (1, n) or (n, 1), to stream ``sid``; staged until the next ``step``"""
        x = np.asarray(block, dtype=np.float32)
        if x.ndim == 2:
            if 1 not in x.shape:
                raise ValueError(f"Waveform must have shape (1, samples) but {x.shape} was found")
            x = x.reshape(-1)
        x = np.ascontiguousarray(x)
        _lib.check(_lib.lib().dg_multi_push_host(self._h, int(sid), x.ctypes.data, len(x)))
        self._pushed[sid] += len(x)

    def available(self, sid: int) -> int:
        n = _lib.lib().dg_multi_available(self._h, int(sid))
        _lib.check(min(n, 0))
        return n

    def window_start_time(self, sid: int, i: int) -> float:
        """start of window i of stream ``sid`` in its output time base (``DeviceAudioStream.window_start_time`` + shift)"""
        return i * self.config.step + float(self._shift[sid])

    def step(self) -> Dict[int, List[Annotation]]:
        """one tick: every open stream's complete windows (at most ``max_windows_per_stream``) -> {sid: annotations}"""
        return self._step()[0]

    def _step(self, outputs: bool = False) -> Tuple[Dict[int, List[Annotation]], Optional[tuple]]:
        """``step``; ``outputs``: also the tick's device outputs (``_outputs``, the handle's ones only), rows grouped by
        stream in slot order"""
        counts = np.where(self._open, np.minimum(available_windows(self._pushed, self._emitted, self._chunk, self._hop),
                                                 self.max_windows_per_stream), 0)
        sids = np.flatnonzero(counts)
        n = counts[sids]
        B = int(n.sum())
        row0 = np.cumsum(n) - n
        idx = np.repeat(self._emitted[sids], n) + (np.arange(B) - np.repeat(row0, n))
        cfg = self.config
        plan, out_start, out_res = mixed_plan(idx, np.repeat(self._latency[sids], n), cfg.step, self.window_samples,
                                              cfg.sample_rate, self.F, self.nw, np.repeat(self._res[sids], n))
        plan = np.ascontiguousarray(plan)
        header = np.empty((B, 4), dtype=np.int32)
        need = turn_capacity(B, self._speakers, self.F)
        if len(self._turns) < need:
            self._turns = np.empty(need, dtype=np.uint32)
        got = np.empty(self.max_streams, dtype=np.int32)
        n_turns = C.c_int()
        outs = self._outputs(B) if outputs and B else (None, None, None)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_multi_step(self._h, plan.ctypes.data, B, got.ctypes.data, header.ctypes.data,
                                                self._turns.ctypes.data, len(self._turns), C.byref(n_turns),
                                                *[_lib.ptr(t) for t in outs]))
        if not np.array_equal(got, counts):
            raise _lib.DiartB200Error("stream bookkeeping out of step with the device handle")
        self._emitted += counts
        self._after_tick(B)
        outs = tuple(t for t in outs if t is not None) or None
        if B == 0:
            return {}, outs
        self._row_sids = np.repeat(sids, n)
        anns = self._annotations(header, self._turns, n_turns.value, out_start, out_res, np.repeat(self._shift[sids], n))
        return {int(s): anns[r:r + k] for s, r, k in zip(sids.tolist(), row0.tolist(), n.tolist())}, outs


class MultiStreamDiarization(_MultiStreamServer):
    """Up to ``max_streams`` live streams diarized on one device with one ``SpeakerDiarizationConfig``:
    ``open(shift, sample_rate) -> sid``, ``push(sid, block)``, ``close(sid)``, and ``step() -> {sid: [Annotation, ...]}`` with
    one ``Annotation`` per window consumed in the tick, in order -- what ``SpeakerDiarization(config)`` returns for that
    stream's windows fed one per call, with its ``timestamp_shift`` set to ``shift``, up to the embedding caveat of the module
    docstring.  A stream is at ``config.sample_rate`` or at one of ``source_sample_rates`` (declared here, see
    ``source_geometry``); its blocks are at its own rate, and its windows are resampled as ``DeviceResample`` resamples them.
    A stream may also have its own ``latency`` (``config.step <= latency <= max_latency``; ``max_latency``, default
    ``config.latency``, at most ``config.duration``, sizes every slot's aggregation history) and ``tau_active``,
    ``rho_update`` and ``delta_new``; its results are then those of ``SpeakerDiarization`` with the config's other values
    and these.  Needs the native models (``B200*Loader``).  ``_step(outputs=True)`` also returns the tick's scores (B, F,
    K), embeddings (B, K, D) and maps (B, K) as device tensors.

    ``open(speakers=known)`` starts a stream from known speakers (:class:`~diart_b200.speakers.KnownSpeakers`, at most
    ``max_speakers`` of the embedding dimension): its results are then those of ``SpeakerDiarization`` with
    ``set_known_speakers(known)``, and its global speaker g < n is labelled ``known.names[g]``.  ``speakers(sid)`` returns the
    stream's active centres with their labels after the last tick; opening a stream with them resumes its clustering state
    exactly (not its aggregation history: the first ``latency / step - 1`` outputs aggregate fewer buffers, as those of any
    new stream do).

    ``gallery`` (a :class:`~diart_b200.speakers.SpeakerGallery` of the embedding dimension; the configuration's metric must
    be cosine): after every tick, each stream that had windows names its active, unnamed global speakers from the gallery by
    the gallery's rule, on the device; the tick's annotations already carry the names it decided, and a name stays for the
    rest of the stream's life.  A stream opened with known speakers counts them as named and their gallery entries as
    claimed, so ``open(speakers=speakers(sid))`` resumes its names and claims.  Names change labels, never segments.

    ``open(gallery=g)`` names that stream from its own gallery ``g`` at ``g.threshold`` for its whole life, whether or not
    the server has a default gallery (``gallery=None``: the server's, if any).  Its names and claims are entries of ``g``,
    so a stream is never named from another stream's gallery, and ``open(speakers=speakers(sid), gallery=g)`` resumes its
    names and claims in ``g``.  Any number of galleries may be in use at once; each tick searches all of them in one grouped
    launch, and a ``SpeakerGallery`` given to many streams is uploaded once.  The server holds each open stream's gallery."""

    _needs = "MultiStreamDiarization needs the native segmentation and embedding models"

    def __init__(self, config: SpeakerDiarizationConfig, max_streams: int, max_windows_per_stream: int = 4,
                 source_sample_rates=(), max_latency: Optional[float] = None, gallery: Optional[SpeakerGallery] = None):
        self._speakers = int(config.max_speakers)
        self.labels = [f"speaker{g}" for g in range(config.max_speakers)]
        self.gallery = gallery
        super().__init__(config, max_streams, max_windows_per_stream, source_sample_rates,
                         (config.segmentation, config.embedding), max_latency)
        if gallery is not None:
            check_gallery(gallery, config, self.D)
            with torch.cuda.device(self.device):
                _lib.check(_lib.lib().dg_multi_set_gallery(self._h, gallery.handle, gallery.threshold))
        self._own_labels = np.zeros(self.max_streams, dtype=bool)      # the slot's labels are its own list, not the shared one
        self._stream_labels = [self.labels] * self.max_streams          # each slot's label list
        # each open slot's gallery (cleared when the slot closes), and whether any stream may be named at all
        self._slot_gallery: List[Optional[SpeakerGallery]] = [None] * self.max_streams
        self._naming = gallery is not None
        self._names = np.empty((0, 3), dtype=np.int32)

    def open(self, shift: float = 0.0, sample_rate: Optional[int] = None, *, latency: Optional[float] = None,
             tau_active: Optional[float] = None, rho_update: Optional[float] = None,
             delta_new: Optional[float] = None, speakers: Optional[KnownSpeakers] = None,
             gallery: Optional[SpeakerGallery] = None) -> int:
        """a new stream in the lowest free slot (``_MultiStreamServer._open_stream``): blocks at ``sample_rate``, time
        stamps shifted by ``shift``, its own latency and thresholds (None: the config's), fixed until it is closed, its
        clustering state seeded with ``speakers`` (None or empty: fresh), and named from ``gallery`` (None: the server's);
        returns its id.  ValueError, with the slot left closed and nothing launched, for known speakers of another
        dimension or more than ``max_speakers`` of them, and for a gallery of another dimension or device (or a
        configuration whose metric is not cosine)."""
        if speakers is not None and not isinstance(speakers, KnownSpeakers):
            raise TypeError(f"speakers: expected KnownSpeakers or None, got {type(speakers).__name__}")
        if gallery is not None:
            check_gallery(gallery, self.config, self.D)
            if not same_device(gallery.device, self.device):
                raise ValueError(f"the gallery is on {gallery.device}, the server on {self.device}")
        known = speakers if speakers is not None and len(speakers) else None
        if known is not None:
            if known.dimension != self.D:
                raise ValueError(f"the known speakers' centroids have dimension {known.dimension}, the embeddings {self.D}")
            if len(known) > self._speakers:
                raise ValueError(f"{len(known)} known speakers, at most max_speakers = {self._speakers}")
        sid = _MultiStreamServer._open_stream(self, shift, sample_rate, latency, None if known is None else known.centroids,
                                              tau_active=tau_active, rho_update=rho_update, delta_new=delta_new)
        gal = self.gallery if gallery is None else gallery
        self._named_by(sid, None if known is None else speaker_labels(known, self._speakers), gal)
        try:
            with torch.cuda.device(self.device):
                if gallery is not None:
                    _lib.check(_lib.lib().dg_multi_set_slot_gallery(self._h, sid, gallery.handle, gallery.threshold))
                if gal is not None and known is not None:
                    named, claimed = gal.claims(self._stream_labels[sid])
                    _lib.check(_lib.lib().dg_multi_set_names(self._h, sid, named, claimed.ctypes.data))
        except BaseException:
            self.close(sid)
            raise
        return sid

    def _named_by(self, sid: int, labels: Optional[List[str]], gallery: Optional[SpeakerGallery]):
        """the labels of the stream that starts in slot ``sid`` (None: the server's) and the gallery it is named from
        (None: none)"""
        self._own_labels[sid] = labels is not None
        self._stream_labels[sid] = self.labels if labels is None else list(labels)
        self._slot_gallery[sid] = gallery
        self._naming = self._naming or gallery is not None

    _kind = "diarization"

    def close(self, sid: int):
        """ends stream ``sid``; the server lets go of its gallery"""
        _MultiStreamServer.close(self, sid)

    def _release(self, sid: int):
        _MultiStreamServer._release(self, sid)
        self._slot_gallery[sid] = None

    def _settings(self) -> dict:
        cfg = self.config
        return dict(_MultiStreamServer._settings(self), D=self.D, max_speakers=int(cfg.max_speakers),
                    gamma=float(cfg.gamma), beta=float(cfg.beta),
                    normalize_embedding_weights=bool(cfg.normalize_embedding_weights),
                    metric=str(getattr(cfg, "metric", "cosine")))

    def _models(self) -> list:
        return _MultiStreamServer._models(self) + [model_fingerprint(self.config.embedding.model)]

    def _stream_meta(self, sid: int) -> dict:
        g = self._slot_gallery[sid]
        return dict(_MultiStreamServer._stream_meta(self, sid),
                    labels=list(self._stream_labels[sid]) if self._own_labels[sid] else None,
                    gallery=None if g is None else gallery_fingerprint(g))

    def _restore_gallery(self, state, gallery):
        want = state._meta["gallery"]
        if want is None:
            return None
        g = self.gallery if gallery is None else gallery
        if g is None:
            raise ValueError("the stream was named from a gallery: give it (gallery=) or serve it as the default")
        if gallery_fingerprint(g) != want:
            raise ValueError("the stream was named from another gallery (names or centroids differ)")
        check_gallery(g, self.config, self.D)
        if not same_device(g.device, self.device):
            raise ValueError(f"the gallery is on {g.device}, the server on {self.device}")
        return g

    def _restored(self, sid, state, gallery):
        _MultiStreamServer._restored(self, sid, state, gallery)
        self._named_by(sid, state._meta["labels"], gallery)

    def speakers(self, sid: int) -> KnownSpeakers:
        """the clustering state of open stream ``sid`` after the last tick: its active centres in index order (a prefix
        0 .. k - 1) with their labels, what ``open(speakers=...)`` resumes from"""
        if not (0 <= sid < self.max_streams and self._open[sid]):
            raise ValueError(f"stream {sid} is not open")
        centers = np.empty((self._speakers, self.D), dtype=np.float64)
        active = np.empty(self._speakers, dtype=np.int32)
        init = C.c_int()
        _lib.check(_lib.lib().dg_multi_get_state(self._h, int(sid), centers.ctypes.data, active.ctypes.data, C.byref(init)))
        return exported(self._stream_labels[sid], centers, active)

    def _create(self, hamming):
        config, emb_net = self.config, self.config.embedding.model
        if not isinstance(emb_net, m.B200XVectorSincNet):
            raise _lib.DiartB200Error(self._needs)
        self.D = emb_net.dims(self.window_samples)[1]
        h = C.c_void_p()
        _lib.check(_lib.lib().dg_multi_create(config.segmentation.model.handle, emb_net.handle, self.window_samples,
                                              self.step_samples, self.max_streams, self.max_windows_per_stream,
                                              int(config.max_speakers), float(config.tau_active), float(config.rho_update),
                                              float(config.delta_new), float(config.gamma), float(config.beta),
                                              int(config.normalize_embedding_weights), self.nw, hamming.ctypes.data,
                                              C.byref(h)))
        return h

    def _outputs(self, B):
        return (torch.empty((B, self.F, self.K), device=self.device), torch.empty((B, self.K, self.D), device=self.device),
                torch.empty((B, self.K), device=self.device, dtype=torch.int32))

    def _after_tick(self, B):
        """the names the tick decided {slot, g, entry} to the slots' labels"""
        if B == 0 or not self._naming:
            return
        n = C.c_int()
        cap = self.max_streams * self._speakers
        if len(self._names) < cap:
            self._names = np.empty((cap, 3), dtype=np.int32)
        _lib.check(_lib.lib().dg_multi_last_names(self._h, self._names.ctypes.data, cap, C.byref(n)))
        for sid, g, e in self._names[:n.value].tolist():
            if not self._own_labels[sid]:
                self._stream_labels[sid] = list(self.labels)
                self._own_labels[sid] = True
            self._stream_labels[sid][g] = self._slot_gallery[sid].names[e]

    def _annotations(self, header, turns, n_turns, out_start, out_res, shifts):
        sids = self._row_sids
        labels = [self._stream_labels[s] for s in sids.tolist()] if self._own_labels[sids].any() else self.labels
        return chunk_annotations(header, turns, n_turns, out_start, out_res, labels, shifts)


class MultiStreamVoiceActivityDetection(_MultiStreamServer):
    """Up to ``max_streams`` live streams through the reference's ``VoiceActivityDetection`` on one device, with the interface
    of ``MultiStreamDiarization``: each window's ``Annotation`` is exactly what ``VoiceActivityDetection(config)`` returns
    for it when the stream is fed one window per call with ``set_timestamp_shift(shift)``.  A tick runs the segmentation
    network alone on all of its windows, then every stream's speech curve (max over the local speakers, aggregated over its
    ``latency / step`` most recent windows) is binarised on the device.  The scores are batch invariant, so a stream's results
    are bit for bit those of its dedicated pipeline whatever the other streams do.  A stream may have its own ``latency``
    (up to ``max_latency``, as ``MultiStreamDiarization``) and ``tau_active``, and is then bit for bit the
    ``VoiceActivityDetection`` at those values.  Needs the native segmentation model (``B200SegmentationLoader``, powerset
    checkpoints included).  ``_step(outputs=True)`` also returns ``(scores,)``, the tick's scores (B, F, K) as a device
    tensor."""

    _needs = "MultiStreamVoiceActivityDetection needs the native segmentation model (B200PyanNet)"
    _speakers = 1
    _kind = "vad"

    def __init__(self, config: VoiceActivityDetectionConfig, max_streams: int, max_windows_per_stream: int = 4,
                 source_sample_rates=(), max_latency: Optional[float] = None, gallery=None):
        if gallery is not None:
            raise ValueError("voice activity detection has no speakers to name: a gallery needs MultiStreamDiarization")
        super().__init__(config, max_streams, max_windows_per_stream, source_sample_rates, (config.segmentation,),
                         max_latency)

    def open(self, shift: float = 0.0, sample_rate: Optional[int] = None, *, latency: Optional[float] = None,
             tau_active: Optional[float] = None, gallery=None) -> int:
        """a new stream in the lowest free slot (``_MultiStreamServer._open_stream``) at its own latency and ``tau_active``
        (None: the config's); returns its id.  ValueError for a ``gallery``: there are no speakers to name"""
        if gallery is not None:
            raise ValueError("voice activity detection has no speakers to name: a gallery needs MultiStreamDiarization")
        return _MultiStreamServer._open_stream(self, shift, sample_rate, latency, tau_active=tau_active)

    def _create(self, hamming):
        h = C.c_void_p()
        _lib.check(_lib.lib().dg_multi_create_vad(self.config.segmentation.model.handle, self.window_samples,
                                                  self.step_samples, self.max_streams, self.max_windows_per_stream,
                                                  float(self.config.tau_active), self.nw, hamming.ctypes.data, C.byref(h)))
        return h

    def _outputs(self, B):
        return torch.empty((B, self.F, self.K), device=self.device), None, None

    def _annotations(self, header, turns, n_turns, out_start, out_res, shifts):
        return speech_annotations(header, turns, n_turns, out_start, out_res, shifts)
