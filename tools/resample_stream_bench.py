"""Measures the device resampler on the GPU and prints one JSON line (and writes it to --out if given):

- the `resample` kernels' time per batch of 256 five-second windows at 44.1 and 48 kHz, stream form (a resampled
  DeviceAudioStream, step 0.5 s) and per-window form (DeviceResample on the stacked source windows);
- SpeakerDiarization.call_stream on a 44.1 kHz stream against the same audio pushed at 16 kHz, in stream-seconds per second;
- the host path the resampled stream replaces: source-rate windows stacked on the host, blocks.Resample on CUDA, __call__.

The networks carry the seeded random weights of oracle/nets.py (timing does not depend on the weight values).  The card's name
and power limit are recorded with the numbers.

    python tools/resample_stream_bench.py [--batches 4] [--out /tmp/resample_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from diart_b200 import blocks, models, synth  # noqa: E402
from diart_b200.blocks.utils import Resample  # noqa: E402
from diart_b200.core import SlidingWindow, SlidingWindowFeature  # noqa: E402
from diart_b200.operators import DeviceAudioStream, DeviceResample  # noqa: E402

B = 256


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [v.strip() for v in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unknown ({e})"
    return info


def cuda_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def kernel_times(src, dev, reps):
    chunk, step = int(round(5 * src)), int(round(0.5 * src))
    audio = np.random.default_rng(src).normal(0, 0.3, chunk + step * (B - 1)).astype(np.float32)
    st = DeviceAudioStream(5, 0.5, 16000, max_windows=B, device=dev, source_sample_rate=src)

    def stream_form():
        st.reset()
        st.push(audio)
        torch.cuda.synchronize()
        t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t[0].record()
        st.windows(B)
        t[1].record()
        torch.cuda.synchronize()
        return t[0].elapsed_time(t[1])

    stream_form()
    stream_ms = float(np.median([stream_form() for _ in range(reps)]))
    rs = DeviceResample(src, 16000, dev)
    x = torch.from_numpy(np.stack([audio[i * step:i * step + chunk] for i in range(B)])).to(dev)
    window_ms = cuda_ms(lambda: rs(x), reps)
    return {"stream_form_ms": stream_ms, "per_window_form_ms": window_ms}


def make_pipe(dev):
    from oracle import nets

    seg, emb = nets.make_segmentation(), nets.make_embedding()
    config = blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg.state_dict())),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb.state_dict())), device=dev)
    return blocks.SpeakerDiarization(config)


def call_stream_rate(src, audio_src, n_batches, dev):
    pipe = make_pipe(dev)
    chunk, step = int(round(5 * src)), int(round(0.5 * src))
    st = DeviceAudioStream(5, 0.5, 16000, max_windows=B, device=dev, source_sample_rate=src)
    st.push(audio_src[:chunk + step * (B - 1)])
    pipe.call_stream(st, B)                                     # warm-up batch
    torch.cuda.synchronize()
    elapsed = 0.0
    for i in range(n_batches):
        lo = chunk + step * (B - 1) + step * B * i
        st.push(audio_src[lo:lo + step * B])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe.call_stream(st, B)
        elapsed += time.perf_counter() - t0
    return n_batches * B * 0.5 / elapsed


def host_path_rate(src, audio_src, n_batches, dev):
    pipe = make_pipe(dev)
    chunk, step = int(round(5 * src)), int(round(0.5 * src))
    resample = Resample(src, 16000, dev)
    sw = SlidingWindow(start=0.0, duration=1 / src, step=1 / src)

    def batch(first):
        out = []
        for i in range(first, first + B):
            w = SlidingWindowFeature(audio_src[i * step:i * step + chunk, None],
                                     SlidingWindow(start=i * 0.5, duration=sw.duration, step=sw.step))
            out.append(resample(w))
        return out

    pipe(batch(0))
    torch.cuda.synchronize()
    elapsed = 0.0
    for i in range(n_batches):
        t0 = time.perf_counter()
        pipe(batch(B * (i + 1)))
        elapsed += time.perf_counter() - t0
    return n_batches * B * 0.5 / elapsed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"card": card(), "windows_per_batch": B}
    for src in (44100, 48000):
        result[f"resample_{src}"] = kernel_times(src, dev, args.reps)
    n16 = 80000 + 8000 * (B * (args.batches + 1) - 1)
    audio16 = synth.synth_audio(n16, seed=9, num_speakers=3)
    audio441 = np.asarray(Resample(16000, 44100, dev)(
        SlidingWindowFeature(audio16[:, None], SlidingWindow(start=0.0, duration=1 / 16000, step=1 / 16000))).data[:, 0],
        dtype=np.float32)
    result["call_stream_16000_stream_s_per_s"] = call_stream_rate(16000, audio16, args.batches, dev)
    result["call_stream_44100_stream_s_per_s"] = call_stream_rate(44100, audio441, args.batches, dev)
    result["host_path_44100_stream_s_per_s"] = host_path_rate(44100, audio441, max(1, args.batches // 2), dev)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
