"""``Binarize`` (mirrors reference ``src/diart/blocks/utils.py:11-59``): discrete-time scores ->
speaker turns at frame middles, label ``speaker<g>`` (or ``labels[g]``)."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from ..core import Annotation, Segment, SlidingWindowFeature


class Binarize:
    def __init__(self, threshold: float, uri: Optional[str] = None, labels: Optional[Sequence[str]] = None):
        self.uri = uri
        self.threshold = threshold
        self.labels = labels          # the label of each global speaker (known speakers' names); None: speaker<g>

    def __call__(self, segmentation: SlidingWindowFeature) -> Annotation:
        num_frames, num_speakers = segmentation.data.shape
        grid = segmentation.sliding_window
        active = segmentation.data > self.threshold
        annotation = Annotation(uri=self.uri, modality="speech")
        lefts = grid.start + grid.step * np.arange(num_frames + 1)
        middles = 0.5 * (lefts + (lefts + grid.duration))        # SlidingWindow[i].middle, as the reference evaluates it
        for spk in np.where(active.any(axis=0))[0]:
            col = np.concatenate([[False], active[:, spk], [False]])
            change = np.flatnonzero(col[1:] != col[:-1])       # on/off boundaries, in frame units
            # a turn that is active from frame 0 starts at the first frame's middle
            for on, off in zip(change[0::2], change[1::2]):
                label = f"speaker{spk}" if self.labels is None else self.labels[spk]
                annotation[Segment(middles[on], middles[off]), int(spk)] = label
        return annotation


class Resample:
    """Resamples audio chunks on the fly (mirrors reference ``src/diart/blocks/utils.py:62-88``; optional pre-processing
    next to the hot path, SURVEY.md 8(f) row 4).  Runs on ``device`` with torchaudio's polyphase resampler."""

    def __init__(self, sample_rate: int, resample_rate: int, device=None):
        import torch
        import torchaudio.transforms as T

        from ..features import TemporalFeatureFormatter

        self.device = torch.device("cpu") if device is None else device
        self.resample = T.Resample(sample_rate, resample_rate).to(self.device)
        self.formatter = TemporalFeatureFormatter()

    def __call__(self, waveform):
        import torch

        wav = self.formatter.cast(waveform).to(self.device)          # (batch, samples, channels)
        with torch.no_grad():
            out = self.resample(wav.transpose(-1, -2)).transpose(-1, -2)
        return self.formatter.restore_type(out)


class AdjustVolume:
    """Scales every chunk to ``volume_in_db`` (10 log10 of the mean power per channel), then divides chunks whose peak would
    exceed 1 by that peak (mirrors reference ``src/diart/blocks/utils.py:91-137``)."""

    def __init__(self, volume_in_db: float):
        from ..features import TemporalFeatureFormatter

        self.target_db = volume_in_db
        self.formatter = TemporalFeatureFormatter()

    @staticmethod
    def get_volumes(waveforms):
        """(batch, samples, channels) -> (batch, 1, channels) volumes in dB"""
        import torch

        return 10 * torch.log10(torch.mean(torch.abs(waveforms) ** 2, dim=1, keepdim=True))

    def __call__(self, waveform):
        import torch

        wav = self.formatter.cast(waveform)
        with torch.no_grad():
            gains = 10 ** ((self.target_db - self.get_volumes(wav)) / 20)
            wav = gains * wav
            peaks = torch.clamp(torch.amax(torch.abs(wav), dim=1, keepdim=True), 1)
            wav = wav / peaks
        return self.formatter.restore_type(wav)
