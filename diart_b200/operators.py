"""Device-side ``rearrange_audio_stream`` (reference ``src/diart/operators.py:44-100``; SURVEY.md 8(f) row 3).

The reference turns an audio stream into 90 %-overlapping windows on the host, so every sample is stacked -- and later
uploaded -- ten times (82 MB per 256-window batch for 8.2 MB of new audio).  ``DeviceAudioStream`` keeps the stream in a
ring buffer in HBM instead: the host pushes each sample once (any block size, like the reference's sources), windows are
formed on the device, and ``SpeakerDiarization.call_stream`` / ``submit_stream`` run the hot path on them.  The host keeps
the same samples in a pinned mirror, from which the aggregated waveform of every output is sliced.

A source at another rate than the pipeline's (a microphone at 44.1 kHz, say) is windowed at the source rate and every window
is resampled to the pipeline's rate on the device, as the reference's ``blocks.Resample`` (torchaudio's ``T.Resample`` with
its defaults) does per window on the host: ``DeviceAudioStream(..., source_sample_rate=44100)``.  ``DeviceResample`` is the
same resampler for device tensors.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib


def sinc_resample_kernel(orig_freq: int, new_freq: int, lowpass_filter_width: int = 6,
                         rolloff: float = 0.99) -> Tuple[np.ndarray, int]:
    """The taps of torchaudio's ``sinc_interp_hann`` resampler, float32 ``(n, 2 width + o)`` for the reduced ratio o / n, and
    ``width``: bit-identical to ``torchaudio.functional.functional._get_sinc_resample_kernel`` (without needing torchaudio).
    As there, the phase offsets ``arange(0, -n, -1) / n`` are float32 and the rest is float64."""
    g = math.gcd(int(orig_freq), int(new_freq))
    o, n = int(orig_freq) // g, int(new_freq) // g
    base = min(o, n) * rolloff
    width = math.ceil(lowpass_filter_width * o / base)
    idx = np.arange(-width, width + o, dtype=np.float64)[None, :] / o
    t = (np.arange(0, -n, -1).astype(np.float32) / np.float32(n))[:, None] + idx
    t = np.clip(t * base, -lowpass_filter_width, lowpass_filter_width)
    window = np.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t = t * math.pi
    with np.errstate(invalid="ignore", divide="ignore"):
        kernel = np.where(t == 0, 1.0, np.sin(t) / t)
    kernel = kernel * (window * (base / o))
    return np.ascontiguousarray(kernel, dtype=np.float32), width


def resample_out_len(orig_freq: int, new_freq: int, num_samples: int) -> int:
    """samples of a resampled ``num_samples``-sample window: ceil(n L / o), in integers (torchaudio evaluates it in float)"""
    g = math.gcd(int(orig_freq), int(new_freq))
    o, n = int(orig_freq) // g, int(new_freq) // g
    return -(-n * int(num_samples) // o)


class DeviceResample:
    """``T.Resample(orig_freq, new_freq)`` (torchaudio defaults) for ``(B, L)`` float32 device tensors, one window per row,
    each zero-padded at its own edges -- what the reference's ``blocks.Resample`` does to every window."""

    def __init__(self, orig_freq: int, new_freq: int, device: Optional[torch.device] = None):
        self.orig_freq, self.new_freq = int(orig_freq), int(new_freq)
        self.device = torch.device(device) if device is not None else torch.device("cuda")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        _lib.require_cuda(self.device)
        self.kernel, self.width = sinc_resample_kernel(self.orig_freq, self.new_freq)
        h = C.c_void_p()
        _lib.check(_lib.lib().dg_resample_create(self.orig_freq, self.new_freq, self.kernel.ctypes.data, self.width,
                                                 self.device.index, C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                _lib.lib().dg_resample_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def out_len(self, num_samples: int) -> int:
        return resample_out_len(self.orig_freq, self.new_freq, num_samples)

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        squeeze = x.dim() == 1
        x = x.reshape(1, -1) if squeeze else x
        if x.dim() != 2 or x.dtype != torch.float32 or x.device != self.device:
            raise ValueError(f"expected a (B, L) float32 tensor on {self.device}, got {tuple(x.shape)} {x.dtype} on {x.device}")
        x = x.contiguous()
        out = torch.empty((x.shape[0], self.out_len(x.shape[1])), device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_resample_forward(self._h, x.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(),
                                                      _lib.stream_ptr(self.device)))
        return out[0] if squeeze else out


class DeviceAudioStream:
    """``sample_rate`` is the pipeline's rate.  ``source_sample_rate`` (default: the same) is the rate of the pushed samples:
    when it differs, the stream is windowed at the source rate (``rearrange_audio_stream(duration, step,
    source_sample_rate)``) and every window is resampled to ``sample_rate`` on the device."""

    def __init__(self, duration: float = 5, step: float = 0.5, sample_rate: int = 16000, max_windows: int = 256,
                 device: Optional[torch.device] = None, start_time: float = 0.0,
                 source_sample_rate: Optional[int] = None):
        self.sample_rate = sample_rate
        self.source_sample_rate = sample_rate if source_sample_rate is None else int(source_sample_rate)
        src = self.source_sample_rate
        self.chunk_samples = int(round(src * duration))      # as operators.py:47-48, at the source rate
        self.step_samples = int(round(src * step))
        self.duration, self.step = duration, step
        self.device = torch.device(device) if device is not None else torch.device("cuda")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        _lib.require_cuda(self.device)
        h = C.c_void_p()
        self.resampler: Optional[DeviceResample] = None
        if src != sample_rate:
            self.resampler = DeviceResample(src, sample_rate, self.device)
            _lib.check(_lib.lib().dg_stream_create_resampled(self.chunk_samples, self.step_samples, self.resampler.handle,
                                                             int(max_windows), self.device.index, C.byref(h)))
        else:
            _lib.check(_lib.lib().dg_stream_create(self.chunk_samples, self.step_samples, int(max_windows),
                                                   self.device.index, C.byref(h)))
        self._h = h
        # samples per window as the pipeline sees them, and their spacing in seconds (the reference's
        # TemporalFeatureFormatter.restore_type after Resample: the source window's duration over the resampled length)
        self.window_samples = self.resampler.out_len(self.chunk_samples) if self.resampler else self.chunk_samples
        self.window_resolution = (self.chunk_samples * (1 / src)) / self.window_samples if self.resampler else 1 / src
        self.start_time = float(start_time)
        self.windows_emitted = 0
        self.audio_stash = {}                   # resampled stream: audio outputs of later chunks, cropped ahead (blocks/post.py)
        # host copy of the not-yet-dropped samples, for the aggregated waveform outputs (audio never comes back from the GPU)
        self._host = np.zeros(0, dtype=np.float32)
        self._host_first = 0                  # absolute index of self._host[0]

    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None:
                _lib.lib().dg_stream_destroy(self._h)
        except Exception:  # noqa: BLE001
            pass

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def push(self, samples: np.ndarray):
        """appends a block of samples: shape (n,), (1, n) (what the reference's sources emit, operators.py:55-58) or (n, 1)"""
        x = np.asarray(samples, dtype=np.float32)
        if x.ndim == 2:
            if 1 not in x.shape:
                raise ValueError(f"Waveform must have shape (1, samples) but {x.shape} was found")
            x = x.reshape(-1)
        x = np.ascontiguousarray(x)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_stream_push_host(self._h, x.ctypes.data, len(x)))
        if self.resampler is None:               # a resampled stream's audio outputs are cropped on the device
            self._host = np.concatenate([self._host, x]) if len(self._host) else x.copy()

    @property
    def available(self) -> int:
        return int(_lib.lib().dg_stream_available(self._h))

    def window_start_time(self, i: int) -> float:
        return self.start_time + i * self.step

    @property
    def resampled(self) -> bool:
        return self.resampler is not None

    def crops(self, ranges) -> np.ndarray:
        """resampled stream: outputs [first, first + count) of window ``window`` for each ``(window, first, count)``, packed in
        one float32 array; the windows must have been formed by the last call and nothing pushed since"""
        r = np.ascontiguousarray(np.asarray(ranges, dtype=np.int64).reshape(-1, 3))
        out = np.empty(int(r[:, 2].sum()), dtype=np.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_stream_crop_host(self._h, len(r), r.ctypes.data, out.ctypes.data))
        return out

    def host_window(self, i: int) -> np.ndarray:
        """window i of the stream from the host copy, shape (chunk_samples, 1)"""
        a = i * self.step_samples - self._host_first
        return self._host[a:a + self.chunk_samples, None]

    def advance(self, n_windows: int, keep_windows: int = 1):
        """bookkeeping after n_windows were consumed: drops host samples no later output can need"""
        self.windows_emitted += n_windows
        first_needed = max(0, self.windows_emitted - keep_windows) * self.step_samples
        if first_needed > self._host_first:
            self._host = self._host[first_needed - self._host_first:]
            self._host_first = first_needed

    def windows(self, n: int) -> torch.Tensor:
        """the next n windows as a dense (n, window_samples) device tensor (consumes them); resampled to ``sample_rate``
        for a source at another rate"""
        out = torch.empty((n, self.window_samples), device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().dg_stream_windows(self._h, n, out.data_ptr(), _lib.stream_ptr(self.device)))
        self.advance(n)
        return out

    def reset(self, start_time: float = 0.0):
        _lib.check(_lib.lib().dg_stream_reset(self._h))
        self.start_time, self.windows_emitted = float(start_time), 0
        self.audio_stash = {}
        self._host, self._host_first = np.zeros(0, dtype=np.float32), 0
