"""Measures tuning VoiceActivityDetection's tau_active over a dataset with VoiceActivitySweep against running the pipeline
once per trial and file (what the reference's Optimizer.objective does) on the GPU, and prints one JSON line (and writes it
to --out if given).

Dataset: the 32 seeded synthetic files of tools/sweep_dataset_bench.py (about 4.8 h), each with its seeded reference.

    construct  VoiceActivitySweep(config, files): the segmentation of every file and the speech curve, once
    sweep      VoiceActivitySweep.score for T in {1, 16, 256, 1024} trials: host clock of the call and CUDA events around
               the launches
    pipeline   for T in {1, 16}: VoiceActivityDetection with each trial's tau_active over every file, Benchmark.run_single's
               way (batches of 256, PredictionAccumulator), scored with oracle/detection.py on the host

The components of the sweep and of the pipeline leg must be equal bit for bit (exit status 1 otherwise).  The card's name
and power limit are recorded with the numbers.

    python tools/vad_sweep_bench.py [--files 32] [--out /tmp/vad_sweep_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from diart_b200 import blocks, models  # noqa: E402
from diart_b200.core import SlidingWindow, SlidingWindowFeature  # noqa: E402
from diart_b200.sinks import PredictionAccumulator  # noqa: E402
from diart_b200.tune import VoiceActivitySweep, file_windows  # noqa: E402
from oracle.detection import detection_components  # noqa: E402
from sweep_bench import card  # noqa: E402
from sweep_dataset_bench import make_dataset  # noqa: E402


def make_config(dev, **kw):
    from oracle import nets

    return blocks.VoiceActivityDetectionConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(nets.make_segmentation().state_dict())),
        device=dev, **kw)


def trials(T, seed=0):
    return [{"tau_active": float(a)} for a in np.random.default_rng(seed + T).uniform(0.2, 0.9, T)]


def pipeline_components(config, files, trials_):
    """one VoiceActivityDetection run per trial and file, scored on the host -> [file] float64 (T, 3)"""
    sr = config.sample_rate
    out = []
    for uri, x, ref in files:
        fw = file_windows(x, config)
        chunks = [SlidingWindowFeature(fw.window(i)[:, None], SlidingWindow(start=fw.starts[i], duration=1 / sr, step=1 / sr))
                  for i in range(fw.num_windows)]
        rows = []
        for trial in trials_:
            config.tau_active = trial["tau_active"]
            pipe = blocks.VoiceActivityDetection(config)
            pipe.set_timestamp_shift(-fw.padding[0])
            acc = PredictionAccumulator(uri)
            for i in range(0, len(chunks), 256):
                for o in pipe(chunks[i:i + 256]):
                    acc.on_next(o)
            rows.append(detection_components(ref, acc.get_prediction()))
        out.append(np.stack(rows))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing to measure")
    dev = torch.device("cuda", 0)
    result = {"card": card()}
    config = make_config(dev)
    files = make_dataset(args.files)
    result["files"] = len(files)
    result["audio_hours"] = sum(len(x) for _, x, _ in files) / 16000 / 3600
    VoiceActivitySweep(config, files[:1]).score(trials(4))          # warm-up: handles, staging, first-use attributes
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    vs = VoiceActivitySweep(config, files)
    result["construct_s"] = time.perf_counter() - t0
    result["construct_parts_s"] = dict(vs.timing)
    result["chunks"] = vs.num_chunks
    result["resident_gb"] = vs.resident_bytes / 1e9
    vs.score(trials(4))                                              # warm-up of the dataset-sized buffers
    rows, equal = {}, True
    for T in (1, 16, 256, 1024):
        tr = trials(T)
        best_call, best_dev = None, None
        for _ in range(3):
            t0 = time.perf_counter()
            got, total = vs.score(tr)
            call = time.perf_counter() - t0
            best_call = call if best_call is None else min(best_call, call)
            best_dev = vs.timing["score"] if best_dev is None else min(best_dev, vs.timing["score"])
        row = {"sweep_score_call_s": best_call, "sweep_score_device_s": best_dev,
               "best_detection_error_rate": float(total.detection_error_rate.min())}
        if T <= 16:
            t0 = time.perf_counter()
            want = pipeline_components(config, files, tr)
            row["pipeline_and_host_score_s"] = time.perf_counter() - t0
            same = all(np.array_equal(g.as_array(), w) for g, w in zip(got, want))
            row["components_equal"] = same
            equal &= same
        rows[T] = row
    result["trials"] = rows
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not equal:
        sys.exit("the sweep's components differ from the pipeline's")


if __name__ == "__main__":
    main()
