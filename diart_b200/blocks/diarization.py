"""``SpeakerDiarization`` pipeline (mirrors reference ``src/diart/blocks/diarization.py:21-234``).

Lines 177-203 of the reference -- segmentation, overlapped-speech penalty, embedding, normalisation
and the sequential clustering loop -- run as ONE fused device step (``dg_pipeline_step``): the
waveform batch is uploaded once, nothing returns to the host in between, and only the
(B,F,K) scores and the (B,K) speaker map come back.  Lines 205-232 (SpeakerMap.apply, aggregation, binarisation) run
on the device too (``blocks/post.py``, ``csrc/post.cu``); the host only attaches time stamps.
"""
from __future__ import annotations

import ctypes as C
import time
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _lib
from .. import models as m
from ..core import Annotation, Segment, SlidingWindow, SlidingWindowFeature, extent_bounds
from ..speakers import KnownSpeakers, exported, speaker_labels
from . import base
from .aggregation import DelayedAggregation
from .clustering import OnlineSpeakerClustering
from .embedding import OverlapAwareSpeakerEmbedding
from .post import DevicePostPath, aggregate_audio, resampled_stream_audio
from .segmentation import SpeakerSegmentation
from .utils import Binarize


class SpeakerDiarizationConfig(base.WindowTiming):
    def __init__(self, segmentation: Optional[m.SegmentationModel] = None,
                 embedding: Optional[m.EmbeddingModel] = None, duration: float = 5, step: float = 0.5,
                 latency=None, tau_active: float = 0.6, rho_update: float = 0.3, delta_new: float = 1,
                 gamma: float = 3, beta: float = 10, max_speakers: int = 20,
                 normalize_embedding_weights: bool = False, device: Optional[torch.device] = None,
                 sample_rate: int = 16000, **kwargs):
        self.segmentation = segmentation or m.SegmentationModel.from_pyannote("pyannote/segmentation")
        self.embedding = embedding or m.EmbeddingModel.from_pyannote("pyannote/embedding")
        self._set_timing(duration, step, latency, sample_rate)
        self.tau_active, self.rho_update, self.delta_new = tau_active, rho_update, delta_new
        self.gamma, self.beta, self.max_speakers = gamma, beta, max_speakers
        self.normalize_embedding_weights = normalize_embedding_weights
        self.device = device or torch.device("cuda")


class SpeakerDiarization(base.Pipeline):
    def __init__(self, config: Optional[SpeakerDiarizationConfig] = None):
        self._config = SpeakerDiarizationConfig() if config is None else config
        msg = f"Latency should be in the range [{self._config.step}, {self._config.duration}]"
        assert self._config.step <= self._config.latency <= self._config.duration, msg
        self.segmentation = SpeakerSegmentation(self._config.segmentation, self._config.device)
        self.embedding = OverlapAwareSpeakerEmbedding(
            self._config.embedding, self._config.gamma, self._config.beta, norm=1,
            normalize_weights=self._config.normalize_embedding_weights, device=self._config.device)
        self.pred_aggregation = DelayedAggregation(self._config.step, self._config.latency,
                                                   strategy="hamming", cropping_mode="loose")
        self.audio_aggregation = DelayedAggregation(self._config.step, self._config.latency,
                                                    strategy="first", cropping_mode="center")
        self.binarize = Binarize(self._config.tau_active)
        self.timestamp_shift = 0
        self.clustering: Optional[OnlineSpeakerClustering] = None
        self.chunk_buffer, self.pred_buffer = [], []
        self._fused: Optional[C.c_void_p] = None
        self._pinned: Optional[torch.Tensor] = None
        self._post: Optional[DevicePostPath] = None
        self.call_profile: Optional[dict] = None       # set to {} to accumulate seconds per phase of __call__
        self._known: Optional[KnownSpeakers] = None
        self.labels = speaker_labels(None, self._config.max_speakers)
        self.reset()

    @staticmethod
    def get_config_class() -> type:
        return SpeakerDiarizationConfig

    @staticmethod
    def suggest_metric():
        from pyannote.metrics.diarization import DiarizationErrorRate  # optional dependency

        return DiarizationErrorRate(collar=0, skip_overlap=False)

    @staticmethod
    def hyper_parameters() -> Sequence[base.HyperParameter]:
        return [base.TauActive, base.RhoUpdate, base.DeltaNew]

    @property
    def config(self) -> SpeakerDiarizationConfig:
        return self._config

    def set_timestamp_shift(self, shift: float):
        self.timestamp_shift = shift

    def reset(self):
        self.set_timestamp_shift(0)
        self._drop_fused()
        self.clustering = OnlineSpeakerClustering(self.config.tau_active, self.config.rho_update,
                                                  self.config.delta_new, "cosine", self.config.max_speakers,
                                                  device=self.segmentation.device)
        self.clustering.seed(None if self._known is None else self._known.centroids)
        self._started = False                          # a chunk went through since construction or reset()
        self.chunk_buffer, self.pred_buffer = [], []
        if self._post is not None:
            self._post.reset()

    # ------------------------------------------------------------------ known speakers
    def set_known_speakers(self, known: Optional[KnownSpeakers]):
        """makes ``known`` the initial clustering state (``diart_b200.speakers``): centres 0 .. n - 1 hold its centroids and
        are active, the state is initialised, and centre g < n is labelled ``names[g]`` in every annotation.  None or an
        empty one: the fresh state.  Only before the first chunk after construction or :meth:`reset`, which re-applies
        it; ValueError otherwise, or for more than ``max_speakers`` speakers.  The dimension is checked against the
        embeddings' before the first clustering launch."""
        if self._started:
            raise ValueError("known speakers are set before the first chunk after construction or reset()")
        if known is not None and not isinstance(known, KnownSpeakers):
            raise TypeError(f"expected KnownSpeakers or None, got {type(known).__name__}")
        known = known if known is not None and len(known) else None
        self.clustering.seed(None if known is None else known.centroids)
        self._known = known
        self.labels = speaker_labels(known, self.config.max_speakers)
        self.binarize.labels = self.labels
        if self._post is not None:
            self._post.labels = self.labels

    def speakers(self) -> KnownSpeakers:
        """the clustering's active centres in index order (a prefix 0 .. k - 1) with their labels: what
        :meth:`set_known_speakers` of a later pipeline resumes from.  The aggregation history is not part of it."""
        if self.clustering._h is None:                # no chunk yet: the initial state
            return self._known if self._known is not None else KnownSpeakers([], np.zeros((0, 0)))
        centers, active, _ = self.clustering._state()
        flags = np.zeros(self.config.max_speakers, dtype=np.int32)
        flags[sorted(active)] = 1
        return exported(self.labels, centers, flags)

    # ------------------------------------------------------------------ fused device step
    def _drop_fused(self):
        if self._fused is not None:
            _lib.lib().dg_pipeline_destroy(self._fused)
            self._fused = None

    def __del__(self):
        try:
            self._drop_fused()
        except Exception:  # noqa: BLE001
            pass

    def _native_models(self):
        seg = getattr(self.segmentation.model, "model", None)
        emb = self.embedding.embedding.native
        scalar_norm = not isinstance(self.embedding.normalize.norm, torch.Tensor)
        if isinstance(seg, m.B200PyanNet) and emb is not None and scalar_norm:
            return seg, emb
        return None

    def _ensure_fused(self, num_samples: int):
        """creates the fused dg_pipeline handle (native models only); returns (handle, F, K, D)"""
        native = self._native_models()
        if native is None:
            raise _lib.DiartB200Error("the fused / pipelined step needs the native segmentation and embedding models")
        seg_net, emb_net = native
        F, K = seg_net.dims(num_samples)
        _, D = emb_net.dims(num_samples)
        if self._fused is None:
            h = C.c_void_p()
            _lib.check(_lib.lib().dg_pipeline_create(seg_net.handle, emb_net.handle, self.clustering._handle(D),
                                                     float(self.config.gamma), float(self.config.beta),
                                                     int(self.config.normalize_embedding_weights), C.byref(h)))
            # consecutive chunks of a batch are `step` seconds apart in one stream (reference operators.py:44-100): a
            # hint for the stream form of the sinc layer; the device verifies it per batch
            _lib.check(_lib.lib().dg_pipeline_set_hop(h, int(round(self.config.step * self.config.sample_rate))))
            self._fused = h
        self._started = True
        return self._fused, F, K, D

    def submit(self, batch: torch.Tensor):
        """Pipelined step (at most three outstanding): enqueue a (B,S) device batch and return; clustering of this step overlaps the
        networks of the next one.  ``batch`` must stay alive until the matching :meth:`collect`."""
        device = self.segmentation.device
        h, F, K, D = self._ensure_fused(batch.shape[1])
        with torch.cuda.device(device):
            _lib.check(_lib.lib().dg_pipeline_submit(h, batch.data_ptr(), batch.shape[0], batch.shape[1],
                                                     _lib.stream_ptr(device)))
        self._pending = getattr(self, "_pending", []) + [(batch.shape[0], F, K, D)]

    def collect(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Oldest submitted step -> (segmentation (B,F,K), embeddings (B,K,D), map (B,K) int32) device tensors
        (copies of the handle's slot buffers, ordered on the current stream)."""
        device = self.segmentation.device
        B, F, K, D = self._pending.pop(0)
        seg = torch.empty((B, F, K), device=device)
        emb = torch.empty((B, K, D), device=device)
        maps = torch.empty((B, K), device=device, dtype=torch.int32)
        with torch.cuda.device(device):
            _lib.check(_lib.lib().dg_pipeline_collect_copy(self._fused, seg.data_ptr(), emb.data_ptr(), maps.data_ptr(),
                                                           _lib.stream_ptr(device)))
        return seg, emb, maps

    def device_step(self, batch: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """batch (B,S) float32 on the device -> (segmentation (B,F,K), embeddings (B,K,D), map (B,K) int32),
        all on the device; clustering state advances by B chunks."""
        native = self._native_models()
        device = self.segmentation.device
        if native is None:  # foreign models behind the loader API: block by block, still on the device
            self._started = True
            seg = self.segmentation.forward_device(batch)
            emb = self.embedding.forward_device(batch, seg)
            maps, _ = self.clustering.step_batch(seg, emb)
            return seg, emb, maps
        B, S = batch.shape
        _, F, K, D = self._ensure_fused(S)
        seg = torch.empty((B, F, K), device=device)
        emb = torch.empty((B, K, D), device=device)
        maps = torch.empty((B, K), device=device, dtype=torch.int32)
        with torch.cuda.device(device):
            _lib.check(_lib.lib().dg_pipeline_step(self._fused, batch.data_ptr(), B, S, seg.data_ptr(),
                                                   emb.data_ptr(), maps.data_ptr(), None, _lib.stream_ptr(device)))
        return seg, emb, maps

    def host_step(self, batch: np.ndarray):
        """batch (B,S) float32 host array -> (segmentation, embeddings, map) numpy arrays; H2D/D2H inside."""
        device = self.segmentation.device
        B, S = batch.shape
        if self._pinned is None or self._pinned.shape != (B, S):
            self._pinned = torch.empty((B, S), dtype=torch.float32).pin_memory()
        self._pinned.copy_(torch.from_numpy(batch))
        dev = self._pinned.to(device, non_blocking=True)
        seg, emb, maps = self.device_step(dev)
        return seg.cpu().numpy(), emb.cpu().numpy(), maps.cpu().numpy()

    # ------------------------------------------------------------------ the pipeline call
    def __call__(self, waveforms: Sequence[SlidingWindowFeature]) -> Sequence[Tuple[Annotation, SlidingWindowFeature]]:
        """reference diarization.py:157-234.  With the native models the whole body is ONE library call
        (``dg_pipeline_call_host``): the B separate host windows are gathered and uploaded by worker threads, the fused
        step and the post-path (aggregation, binarisation, run-length turns) run on the device, and only the packed turn
        list returns; the host attaches time stamps."""
        batch_size = len(waveforms)
        assert batch_size >= 1, "Pipeline expected at least 1 input"
        expected = int(np.rint(self.config.duration * self.config.sample_rate))
        if self._native_models() is None:
            return self._call_blockwise(waveforms, expected)
        prof = self.call_profile          # None, or a dict of accumulated seconds per phase (bench.py)
        t0 = time.perf_counter() if prof is not None else 0.0
        rows, f32 = [], np.float32
        for w in waveforms:
            d = w.data
            shape = d.shape
            assert shape[0] == expected, f"Expected {expected} samples per chunk, but got {shape[0]}"
            assert len(shape) == 1 or shape[1] == 1, "expected mono audio"
            if d.dtype != f32 or not d.flags.c_contiguous:
                d = np.ascontiguousarray(d, dtype=f32)
            rows.append(d)
        h, F, K, D = self._ensure_fused(expected)
        post = self._ensure_post(F, K)
        starts = np.array([extent_bounds(w)[0] for w in waveforms], dtype=np.float64)
        seg_resolution = waveforms[0].extent.duration / F
        plan, out_start, out_res = post.plan(starts, seg_resolution)
        header, turns = post.buffers(batch_size)
        ptrs = (C.c_void_p * batch_size)(*[r.__array_interface__["data"][0] for r in rows])
        n_turns = C.c_int()
        t1 = time.perf_counter() if prof is not None else 0.0
        with torch.cuda.device(self.segmentation.device):
            _lib.check(_lib.lib().dg_pipeline_call_host(h, post.handle, ptrs, batch_size, expected, plan.ctypes.data,
                                                        header.ctypes.data, turns.ctypes.data, len(turns),
                                                        C.byref(n_turns), None, None))
        t2 = time.perf_counter() if prof is not None else 0.0
        annotations = post.annotations(header, turns, n_turns.value, out_start, out_res, self.timestamp_shift)
        t3 = time.perf_counter() if prof is not None else 0.0
        audio, self.chunk_buffer = aggregate_audio(self.chunk_buffer, waveforms, post.nw, self.config.step,
                                                   self.config.latency)
        out = list(zip(annotations, audio))
        if prof is not None:
            t4 = time.perf_counter()
            for key, dt in (("prepare", t1 - t0), ("library_call", t2 - t1), ("annotations", t3 - t2), ("audio", t4 - t3)):
                prof[key] = prof.get(key, 0.0) + dt
            prof["calls"] = prof.get("calls", 0) + 1
        return out

    def call_stream(self, stream, batch_size: Optional[int] = None):
        """``__call__`` for the next ``batch_size`` windows (default: all available) of a
        :class:`diart_b200.operators.DeviceAudioStream`: the windows never exist on the host, only each new sample was
        uploaded once.  Returns the same ``[(Annotation, SlidingWindowFeature), ...]`` as ``__call__`` on the windows
        ``rearrange_audio_stream`` would have emitted.

        A stream at another source rate is resampled on the device (reference: ``blocks.Resample`` after
        ``rearrange_audio_stream(source_rate)``); the result is then ``__call__`` on the resampled windows with the
        reference's time base, and the audio outputs are crops of the resampled windows, of which only the cropped ranges
        return to the host."""
        B = stream.available if batch_size is None else int(batch_size)
        assert B >= 1, "Pipeline expected at least 1 input"
        expected = int(np.rint(self.config.duration * self.config.sample_rate))
        if getattr(stream, "resampled", False):
            assert stream.sample_rate == self.config.sample_rate, \
                f"the stream resamples to {stream.sample_rate} Hz, the pipeline runs at {self.config.sample_rate} Hz"
            return self._call_resampled_stream(stream, B, expected)
        assert stream.chunk_samples == expected, f"Expected {expected} samples per chunk, but got {stream.chunk_samples}"
        if self._native_models() is None:
            raise _lib.DiartB200Error("call_stream needs the native segmentation and embedding models")
        h, F, K, D = self._ensure_fused(expected)
        post = self._ensure_post(F, K)
        sr = stream.sample_rate
        first = stream.windows_emitted
        sws = [SlidingWindow(start=stream.window_start_time(first + i), duration=1 / sr, step=1 / sr) for i in range(B)]
        waves = [SlidingWindowFeature(stream.host_window(first + i), sw) for i, sw in enumerate(sws)]
        starts = np.array([w.extent.start for w in waves], dtype=np.float64)
        plan, out_start, out_res = post.plan(starts, waves[0].extent.duration / F)
        header, turns = post.buffers(B)
        n_turns = C.c_int()
        with torch.cuda.device(self.segmentation.device):
            _lib.check(_lib.lib().dg_pipeline_call_stream(h, post.handle, stream.handle, B, plan.ctypes.data,
                                                          header.ctypes.data, turns.ctypes.data, len(turns),
                                                          C.byref(n_turns), None, None))
        annotations = post.annotations(header, turns, n_turns.value, out_start, out_res, self.timestamp_shift)
        audio, self.chunk_buffer = aggregate_audio(self.chunk_buffer, waves, post.nw, self.config.step, self.config.latency)
        stream.advance(B, keep_windows=post.nw)
        return list(zip(annotations, audio))

    def _call_resampled_stream(self, stream, B: int, expected: int):
        """call_stream on a stream whose windows are resampled on the device (see call_stream)"""
        n = stream.window_samples
        assert n == expected, f"Expected {expected} samples per chunk, but got {n}"
        if self._native_models() is None:
            raise _lib.DiartB200Error("call_stream needs the native segmentation and embedding models")
        h, F, K, D = self._ensure_fused(expected)
        post = self._ensure_post(F, K)
        first = stream.windows_emitted
        starts = np.array([stream.window_start_time(first + i) for i in range(B)], dtype=np.float64)
        res = stream.window_resolution
        s0, e0 = starts[0], starts[0] + n * res                           # extent of the first window
        plan, out_start, out_res = post.plan(starts, (e0 - s0 if e0 > s0 else 0.0) / F)
        header, turns = post.buffers(B)
        n_turns = C.c_int()
        with torch.cuda.device(self.segmentation.device):
            _lib.check(_lib.lib().dg_pipeline_call_stream(h, post.handle, stream.handle, B, plan.ctypes.data,
                                                          header.ctypes.data, turns.ctypes.data, len(turns),
                                                          C.byref(n_turns), None, None))
        annotations = post.annotations(header, turns, n_turns.value, out_start, out_res, self.timestamp_shift)
        audio = resampled_stream_audio(stream, first, B, post.nw, self.config.step, self.config.latency)
        stream.advance(B, keep_windows=post.nw)
        return list(zip(annotations, audio))

    def _ensure_post(self, F: int, K: int) -> DevicePostPath:
        if self._post is None:
            self._post = DevicePostPath(self.config.step, self.config.latency, self.config.tau_active, F, K,
                                        self.config.max_speakers, self.segmentation.device)
            self._post.labels = self.labels
        return self._post

    def _call_blockwise(self, waveforms, expected):
        """foreign models behind the loader API: block by block, host-side aggregation (numpy mirrors of the reference)"""
        batch = np.stack([np.asarray(w.data, dtype=np.float32) for w in waveforms])   # (batch, samples, channels)
        assert batch.shape[1] == expected, f"Expected {expected} samples per chunk, but got {batch.shape[1]}"
        assert batch.shape[2] == 1, "expected mono audio"
        seg, _, maps = self.host_step(np.ascontiguousarray(batch[:, :, 0]))
        num_frames = seg.shape[1]
        seg_resolution = waveforms[0].extent.duration / num_frames
        outputs = []
        for wav, s, amap in zip(waveforms, seg, maps):
            sw = SlidingWindow(start=wav.extent.start, duration=seg_resolution, step=seg_resolution)
            permuted = np.zeros((num_frames, self.config.max_speakers))          # SpeakerMap.apply
            for k, g in enumerate(amap):
                if g >= 0:
                    permuted[:, g] = s[:, k]
            self.chunk_buffer.append(wav)
            self.pred_buffer.append(SlidingWindowFeature(permuted, sw))
            agg_waveform = self.audio_aggregation(self.chunk_buffer)
            agg_prediction = self.binarize(self.pred_aggregation(self.pred_buffer))
            if self.timestamp_shift != 0:
                shifted = Annotation(agg_prediction.uri)
                for segment, track, speaker in agg_prediction.itertracks(yield_label=True):
                    shifted[Segment(segment.start + self.timestamp_shift,
                                    segment.end + self.timestamp_shift), track] = speaker
                agg_prediction = shifted
            outputs.append((agg_prediction, agg_waveform))
            if len(self.chunk_buffer) == self.pred_aggregation.num_overlapping_windows:
                self.chunk_buffer = self.chunk_buffer[1:]
                self.pred_buffer = self.pred_buffer[1:]
        return outputs
