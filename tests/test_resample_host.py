"""Host half of the device resampler (csrc/resample.cu, diart_b200.operators): the tap table is torchaudio's bit for bit, the
float64 oracle of the polyphase convolution agrees with torchaudio, the output length follows torchaudio's rule, the C ABI
rejects bad tap tables without touching a GPU, and the audio crops of a resampled stream equal aggregate_audio's."""
import ctypes as C
import math

import numpy as np
import pytest

from diart_b200 import _lib
from diart_b200.blocks.post import aggregate_audio, resampled_stream_audio
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.operators import resample_out_len, sinc_resample_kernel

PAIRS = [(8000, 16000), (11025, 16000), (22050, 16000), (24000, 16000), (32000, 16000), (44100, 16000), (48000, 16000),
         (16000, 8000)]


def oracle_resample(x: np.ndarray, kernel: np.ndarray, orig: int, new: int, width: int) -> np.ndarray:
    """float64 restatement of torchaudio's _apply_sinc_resample_kernel: x (B, L) zero-padded by (width, width + o), strided
    by o, one output per phase, truncated to ceil(n L / o)"""
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    x = np.atleast_2d(np.asarray(x, dtype=np.float64))
    L = x.shape[1]
    xp = np.pad(x, ((0, 0), (width, width + o)))
    frames = np.lib.stride_tricks.sliding_window_view(xp, kernel.shape[1], axis=1)[:, ::o]   # (B, L // o + 1, T)
    y = frames @ np.asarray(kernel, dtype=np.float64).T                                     # (B, frames, n)
    return y.reshape(x.shape[0], -1)[:, :resample_out_len(orig, new, L)]


@pytest.mark.parametrize("orig,new", PAIRS)
def test_taps_are_torchaudios_bit_for_bit(orig, new):
    ta = pytest.importorskip("torchaudio.functional.functional")
    ref, width = ta._get_sinc_resample_kernel(orig, new, math.gcd(orig, new))
    taps, w = sinc_resample_kernel(orig, new)
    assert w == width
    assert taps.dtype == np.float32 and taps.shape == tuple(ref[:, 0].shape)
    assert np.array_equal(taps.view(np.uint32), ref[:, 0].numpy().view(np.uint32))


@pytest.mark.parametrize("orig,new", [(44100, 16000), (48000, 16000), (8000, 16000), (11025, 16000)])
def test_float64_oracle_matches_torchaudio(orig, new):
    torch = pytest.importorskip("torch")
    taf = pytest.importorskip("torchaudio.functional")
    rng = np.random.default_rng(orig)
    x = rng.normal(0, 0.3, (3, 3 * orig // 4 + 17))
    want = taf.resample(torch.from_numpy(x), orig, new).numpy()            # float64 end to end (float64 taps)
    from torchaudio.functional.functional import _get_sinc_resample_kernel

    k64, width = _get_sinc_resample_kernel(orig, new, math.gcd(orig, new), dtype=torch.float64)
    got = oracle_resample(x, k64[:, 0].numpy(), orig, new, width)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-12


@pytest.mark.parametrize("orig,new", [(44100, 16000), (48000, 16000), (8000, 16000), (11025, 16000), (16000, 8000)])
def test_output_length_rule_matches_torchaudio(orig, new):
    torch = pytest.importorskip("torch")
    taf = pytest.importorskip("torchaudio.functional")
    g = math.gcd(orig, new)
    o = orig // g
    lengths = [L for L in (1, 2 * o - 1, o + 1, 5 * o + 1, 220501, 240001, 80007) if L % o or o == 1]
    assert len(lengths) >= 5
    for L in lengths:
        got = resample_out_len(orig, new, L)
        assert got == taf.resample(torch.zeros(1, L), orig, new).shape[-1], L


def test_resample_create_rejects_bad_taps_without_a_gpu():
    lib = _lib.lib()
    taps, width = sinc_resample_kernel(44100, 16000)
    h = C.c_void_p()
    assert lib.dg_resample_create(44100, 16000, taps.ctypes.data, width + 1, 0, C.byref(h)) == -1   # (160, 477) table
    assert "expected" in lib.dg_last_error().decode()
    assert lib.dg_resample_create(48000, 16000, taps.ctypes.data, width, 0, C.byref(h)) == -1       # 44.1k taps for 48k
    assert lib.dg_resample_create(0, 16000, taps.ctypes.data, width, 0, C.byref(h)) == -1
    assert lib.dg_resample_create(44100, -16000, taps.ctypes.data, width, 0, C.byref(h)) == -1
    assert lib.dg_resample_create(16000, 16000, taps.ctypes.data, width, 0, C.byref(h)) == -1
    assert lib.dg_resample_create(44100, 16000, None, width, 0, C.byref(h)) == -1
    assert lib.dg_resample_out_len(None, 100) == -1
    assert lib.dg_stream_create_resampled(220500, 22050, None, 8, 0, C.byref(h)) == -1
    assert lib.dg_stream_crop_host(None, 0, None, None) == -1


class _FakeResampledStream:
    """the host-visible surface of a resampled DeviceAudioStream, its windows held in numpy"""

    def __init__(self, windows: np.ndarray, src_rate: int, chunk_src: int, step: float, start_time: float = 0.0):
        self.w = windows
        self.window_samples = windows.shape[1]
        self.window_resolution = (chunk_src * (1 / src_rate)) / self.window_samples
        self.step, self.start_time = step, start_time
        self.audio_stash = {}
        self.fetched = 0

    def window_start_time(self, i):
        return self.start_time + i * self.step

    def crops(self, ranges):
        self.fetched += sum(k for _, _, k in ranges)
        return np.concatenate([self.w[o, a:a + k] for o, a, k in ranges]).astype(np.float32)


@pytest.mark.parametrize("latency,batches", [(1.5, [7, 1, 12, 5]), (0.5, [3, 4]), (5.0, [2, 11, 20])])
def test_resampled_stream_audio_equals_aggregate_audio(latency, batches):
    step, duration, src = 0.5, 5.0, 44100
    chunk_src = int(round(src * duration))
    L = resample_out_len(src, 16000, chunk_src)
    total = sum(batches)
    rng = np.random.default_rng(3)
    windows = rng.normal(0, 0.3, (total, L)).astype(np.float32)
    fake = _FakeResampledStream(windows, src, chunk_src, step)
    nw = int(round(latency / step))
    res = fake.window_resolution
    buf, first = [], 0
    for B in batches:
        waves = [SlidingWindowFeature(windows[i, :, None], SlidingWindow(start=fake.window_start_time(i), duration=res, step=res))
                 for i in range(first, first + B)]
        want, buf = aggregate_audio(buf, waves, nw, step, latency)
        got = resampled_stream_audio(fake, first, B, nw, step, latency)
        for c, (a, b) in enumerate(zip(want, got)):
            assert np.array_equal(a.data, b.data), f"chunk {first + c}"
            sa, sb = a.sliding_window, b.sliding_window
            assert (sa.start, sa.duration, sa.step) == (sb.start, sb.duration, sb.step), f"chunk {first + c}"
        first += B
    assert fake.fetched < total * L / 4          # crops only, not whole windows
