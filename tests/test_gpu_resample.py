"""Device resampling (csrc/resample.cu): the per-window form against a float64 oracle and torchaudio, the stream form of a
resampled DeviceAudioStream bit-identical to the per-window form on the stacked source windows, and the pipeline on a
44.1 / 48 kHz stream identical to the pipeline on the resampled windows."""
import numpy as np
import pytest
import torch

from diart_b200 import _lib, synth
from diart_b200.core import SlidingWindow, SlidingWindowFeature
from diart_b200.operators import DeviceAudioStream, DeviceResample
from test_gpu_pipeline import make_pipeline
from test_resample_host import oracle_resample

pytestmark = pytest.mark.gpu


def source_audio(n_samples: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return np.clip(rng.normal(0, 0.3, n_samples), -1, 1).astype(np.float32)


def stacked(audio: np.ndarray, chunk: int, step: int, n: int, first: int = 0) -> np.ndarray:
    return np.stack([audio[(first + i) * step:(first + i) * step + chunk] for i in range(n)])


@pytest.mark.parametrize("orig", [44100, 48000, 8000, 11025])
@pytest.mark.parametrize("B,L", [(1, 220501), (7, 44107), (256, 9001)])
def test_per_window_form_against_float64_oracle_and_torchaudio(cuda_device, orig, B, L):
    rs = DeviceResample(orig, 16000, cuda_device)
    x = np.stack([source_audio(L, 11 * b + orig) for b in range(B)])
    got = rs(torch.from_numpy(x).to(cuda_device)).cpu().numpy()
    want = oracle_resample(x, rs.kernel, orig, 16000, rs.width)
    assert got.shape == want.shape == (B, rs.out_len(L))
    assert np.abs(got - want).max() <= 1e-6
    ta = pytest.importorskip("torchaudio.transforms")
    ref = ta.Resample(orig, 16000)(torch.from_numpy(x)).numpy()
    assert np.abs(got - ref).max() <= 1.5e-6


@pytest.mark.parametrize("src,step", [(44100, 0.5), (48000, 0.5), (8000, 0.5), (44100, 0.125)])
def test_stream_windows_equal_per_window_form_on_stacked_windows(cuda_device, src, step):
    """stream form (step % o == 0) and per-window form from the ring (44.1 kHz at 0.125 s): ragged pushes, ring wrap-around"""
    st = DeviceAudioStream(5, step, 16000, max_windows=16, device=cuda_device, source_sample_rate=src)
    assert st.chunk_samples == int(round(5 * src)) and st.window_samples == 80000
    rs = DeviceResample(src, 16000, cuda_device)
    n = 70
    audio = source_audio(st.chunk_samples + st.step_samples * (n - 1), seed=src)
    rng = np.random.default_rng(1)
    pos, emitted = 0, 0
    while emitted < n:
        while st.available < min(16, n - emitted) and pos < len(audio):
            k = int(rng.integers(1, st.step_samples * 3))
            st.push(audio[pos:pos + k])
            pos += k
        b = min(st.available, int(rng.integers(1, 17)), n - emitted)
        got = st.windows(b).cpu().numpy()
        x = stacked(audio, st.chunk_samples, st.step_samples, b, emitted)
        want = rs(torch.from_numpy(x).to(cuda_device)).cpu().numpy()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"windows {emitted}..{emitted + b}"
        # crops of the windows just formed are the same bits
        crop = st.crops([(emitted, 0, 300), (emitted + b - 1, 79500, 500)])
        assert np.array_equal(crop, np.concatenate([want[0, :300], want[-1, 79500:]]))
        emitted += b
    assert pos > st.step_samples * 16 * 2          # the ring wrapped around


def resampled_windows(rs, audio, chunk, step, n, start_time, step_s, src):
    """the reference's windows: rearrange_audio_stream at the source rate, Resample, TemporalFeatureFormatter time base"""
    x = rs(torch.from_numpy(stacked(audio, chunk, step, n)).to(rs.device)).cpu().numpy()
    res = (chunk * (1 / src)) / x.shape[1]
    return x, [SlidingWindowFeature(x[i, :, None], SlidingWindow(start=start_time + i * step_s, duration=res, step=res))
               for i in range(n)]


@pytest.mark.parametrize("src", [44100, 48000])
def test_pipeline_on_a_resampled_stream_equals_pipeline_on_resampled_windows(oracle_nets, cuda_device, src):
    n, step_s = 40, 0.5
    chunk, step = int(round(5 * src)), int(round(step_s * src))
    audio = synth.synth_audio(80000 + 8000 * (n - 1), seed=77, num_speakers=3)
    # the synthetic stream at the source rate (any band-limited signal serves)
    ta = pytest.importorskip("torchaudio.transforms")
    audio = ta.Resample(16000, src)(torch.from_numpy(audio)).numpy().astype(np.float32)[:chunk + step * (n - 1)]
    rs = DeviceResample(src, 16000, cuda_device)
    x, waves = resampled_windows(rs, audio, chunk, step, n, 0.0, step_s, src)

    a, b = make_pipeline(oracle_nets, cuda_device, latency=1.5), make_pipeline(oracle_nets, cuda_device, latency=1.5)
    want = a(waves[:17]) + a(waves[17:])
    st = DeviceAudioStream(5, step_s, 16000, max_windows=24, device=cuda_device, source_sample_rate=src)
    st.push(audio[:chunk + step * 16])
    got = b.call_stream(st)
    st.push(audio[chunk + step * 16:])
    got += b.call_stream(st, 23)
    assert len(got) == n
    for i, ((a1, w1), (a2, w2)) in enumerate(zip(want, got)):
        assert a1.to_rttm() == a2.to_rttm(), f"chunk {i}"
        assert np.array_equal(w1.data, w2.data), f"chunk {i}"
        s1, s2 = w1.sliding_window, w2.sliding_window
        assert (s1.start, s1.duration, s1.step) == (s2.start, s2.duration, s2.step), f"chunk {i}"
    assert np.array_equal(a.clustering.centers, b.clustering.centers)

    # pipelined form through the C ABI == dg_pipeline_step_host on the resampled windows
    lib = _lib.lib()
    c, d = make_pipeline(oracle_nets, cuda_device), make_pipeline(oracle_nets, cuda_device)
    hc, F, K, D = c._ensure_fused(80000)
    hd = d._ensure_fused(80000)[0]
    st2 = DeviceAudioStream(5, step_s, 16000, max_windows=40, device=cuda_device, source_sample_rate=src)
    st2.push(audio)
    outs = []
    for i in range(2):
        _lib.check(lib.dg_pipeline_submit_stream(hc, st2.handle, 20))
    for i in range(2):
        s, e, m = np.empty((20, F, K), np.float32), np.empty((20, K, D), np.float32), np.empty((20, K), np.int32)
        _lib.check(lib.dg_pipeline_collect_host(hc, s.ctypes.data, e.ctypes.data, m.ctypes.data))
        outs.append((s, e, m))
    scores = []
    for i in range(2):
        xi = np.ascontiguousarray(x[20 * i:20 * i + 20])
        s, e, m = np.empty((20, F, K), np.float32), np.empty((20, K, D), np.float32), np.empty((20, K), np.int32)
        _lib.check(lib.dg_pipeline_step_host(hd, xi.ctypes.data, 20, 80000, s.ctypes.data, e.ctypes.data, m.ctypes.data, None))
        assert np.array_equal(s, outs[i][0]) and np.array_equal(e, outs[i][1]) and np.array_equal(m, outs[i][2]), f"batch {i}"
        scores.append(s)

    # the same pipeline fed with torchaudio-resampled windows (float32 on the CPU) agrees to 1e-4
    f = make_pipeline(oracle_nets, cuda_device)
    hf = f._ensure_fused(80000)[0]
    xt = ta.Resample(src, 16000)(torch.from_numpy(stacked(audio, chunk, step, n))).numpy()
    for i in range(2):
        xi = np.ascontiguousarray(xt[20 * i:20 * i + 20], dtype=np.float32)
        s, e, m = np.empty((20, F, K), np.float32), np.empty((20, K, D), np.float32), np.empty((20, K), np.int32)
        _lib.check(lib.dg_pipeline_step_host(hf, xi.ctypes.data, 20, 80000, s.ctypes.data, e.ctypes.data, m.ctypes.data, None))
        assert np.abs(s - scores[i]).max() <= 1e-4, f"batch {i}"
