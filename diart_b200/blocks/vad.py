"""``VoiceActivityDetection`` pipeline (reference ``src/diart/blocks/vad.py:27-191``; SURVEY.md 8(f) row 4): the segmentation
network of the hot path, a max over the local speakers, and the same device post-path as the diarization pipeline
(Hamming-weighted aggregation over the ``latency / step`` most recent chunks, threshold, run-length turns: ``csrc/post.cu``)
with ONE "speaker" whose turns are labelled ``"speech"``."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import models as m
from ..core import Annotation, Segment, SlidingWindowFeature
from . import base
from .post import DevicePostPath, aggregate_audio, chunk_turns
from .segmentation import SpeakerSegmentation


def speech_annotations(header: np.ndarray, turns: np.ndarray, n_turns: int, out_start: np.ndarray, out_res: np.ndarray,
                       shift=0.0) -> List[Annotation]:
    """the device post-path's turns of one speaker (``header`` (B, 4), packed ``turns``, as ``chunk_annotations`` takes them)
    -> what ``VoiceActivityDetection`` returns per chunk: tracks numbered in order, label ``"speech"``, modality ``"speech"``
    (reference vad.py:172-178).  A chunk's turns come in time order and do not overlap, so their order is the tracks' order.
    ``shift``: one number, or one per chunk."""
    offs, cnts, _, t_on, t_off = chunk_turns(header, turns, n_turns, out_start, out_res, shift)
    outputs = []
    for o, k in zip(offs, cnts):
        speech = Annotation(modality="speech")
        for n, i in enumerate(range(o, o + k)):
            speech[Segment(t_on[i], t_off[i]), n] = "speech"
        outputs.append(speech)
    return outputs


class VoiceActivityDetectionConfig(base.WindowTiming):
    def __init__(self, segmentation: Optional[m.SegmentationModel] = None, duration: float = 5, step: float = 0.5,
                 latency=None, tau_active: float = 0.6, device: Optional[torch.device] = None,
                 sample_rate: int = 16000, **kwargs):
        self.segmentation = segmentation or m.SegmentationModel.from_pyannote("pyannote/segmentation")
        self._set_timing(duration, step, latency, sample_rate)
        self.tau_active = tau_active
        self.device = device or torch.device("cuda")


class VoiceActivityDetection(base.Pipeline):
    def __init__(self, config: Optional[VoiceActivityDetectionConfig] = None):
        self._config = config if config is not None else VoiceActivityDetectionConfig()
        lo, hi = self._config.step, self._config.duration
        assert lo <= self._config.latency <= hi, f"Latency should be in the range [{lo}, {hi}]"
        self.segmentation = SpeakerSegmentation(self._config.segmentation, self._config.device)
        self.timestamp_shift = 0
        self.chunk_buffer = []
        self._post: Optional[DevicePostPath] = None

    get_config_class = staticmethod(lambda: VoiceActivityDetectionConfig)
    hyper_parameters = staticmethod(lambda: [base.TauActive])

    @staticmethod
    def suggest_metric():
        from pyannote.metrics.detection import DetectionErrorRate  # optional dependency

        return DetectionErrorRate(collar=0, skip_overlap=False)

    @property
    def config(self) -> VoiceActivityDetectionConfig:
        return self._config

    def set_timestamp_shift(self, shift: float):
        self.timestamp_shift = shift

    def reset(self):
        self.set_timestamp_shift(0)
        self.chunk_buffer = []
        if self._post is not None:
            self._post.reset()

    def __call__(self, waveforms: Sequence[SlidingWindowFeature]) -> Sequence[Tuple[Annotation, SlidingWindowFeature]]:
        B, cfg = len(waveforms), self._config
        assert B >= 1, "Pipeline expected at least 1 input"
        expected = int(np.rint(cfg.duration * cfg.sample_rate))
        for w in waveforms:
            assert w.data.shape[0] == expected, f"Expected {expected} samples per chunk, but got {w.data.shape[0]}"
        batch = torch.from_numpy(np.stack([np.asarray(w.data, dtype=np.float32) for w in waveforms]))
        scores = self.segmentation.forward_device(batch)                  # (B, frames, local speakers), stays on the device
        vad = scores.amax(dim=-1, keepdim=True).contiguous()              # reference vad.py:145-148
        F, device = vad.shape[1], vad.device
        if self._post is None:
            self._post = DevicePostPath(cfg.step, cfg.latency, cfg.tau_active, F, 1, 1, device)
        starts = np.array([w.extent.start for w in waveforms], dtype=np.float64)
        to_first = torch.zeros((B, 1), dtype=torch.int32, device=device)  # the one local "speaker" is global speaker 0
        outputs = speech_annotations(*self._post.turns(vad, to_first, starts, waveforms[0].extent.duration / F),
                                     self.timestamp_shift)
        audio, self.chunk_buffer = aggregate_audio(self.chunk_buffer, waveforms, self._post.nw, cfg.step, cfg.latency)
        return list(zip(outputs, audio))
