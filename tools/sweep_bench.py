"""Measures the hyper-parameter sweep (diart_b200.tune) on the GPU and prints one JSON line (and writes it to --out if given).

Input: a seeded synthetic 30-minute file (synth.synth_audio) at the default config.  For T in {1, 16, 64, 256} trials:
- the network pass (once per file, fused pipeline in batches of 256),
- dg_sweep_run (clustering + post-path of all T trials; CUDA events around the synchronous call),
- the host assembly of the T whole-file predictions,
each separately; and, for T = 16 only, the baseline the sweep replaces: T sequential SpeakerDiarization runs over the same
windows (batches of 256, PredictionAccumulator), whose predictions are checked to equal the sweep's.  The networks carry the
seeded random weights of oracle/nets.py (timing does not depend on the weight values).  The card's name and power limit are
recorded with the numbers.

    python tools/sweep_bench.py [--minutes 30] [--out /tmp/sweep_bench.json]
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
from diart_b200.core import SlidingWindow, SlidingWindowFeature  # noqa: E402
from diart_b200.sinks import PredictionAccumulator  # noqa: E402
from diart_b200.tune import HyperParameterSweep, file_windows, trial_params  # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [v.strip() for v in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unknown ({e})"
    return info


def make_config(dev, **kw):
    from oracle import nets

    seg, emb = nets.make_segmentation(), nets.make_embedding()
    return blocks.SpeakerDiarizationConfig(
        segmentation=models.SegmentationModel(models.B200SegmentationLoader(seg.state_dict())),
        embedding=models.EmbeddingModel(models.B200EmbeddingLoader(emb.state_dict())), device=dev, **kw)


def trials(T, seed=0):
    rng = np.random.default_rng(seed + T)
    return [{"tau_active": float(a), "rho_update": float(b), "delta_new": float(c)}
            for a, b, c in zip(rng.uniform(0.3, 0.8, T), rng.uniform(0, 1, T), rng.uniform(0.1, 2, T))]


def baseline(config, fw, params, uri):
    """one SpeakerDiarization run per trial, Benchmark.run_single's way -> (predictions, seconds per run)"""
    sr = config.sample_rate
    chunks = [SlidingWindowFeature(fw.window(i)[:, None], SlidingWindow(start=fw.starts[i], duration=1 / sr, step=1 / sr))
              for i in range(fw.num_windows)]
    preds, secs = [], []
    for tau, rho, delta in params:
        c = blocks.SpeakerDiarizationConfig(segmentation=config.segmentation, embedding=config.embedding,
                                            device=config.device, tau_active=tau, rho_update=rho, delta_new=delta)
        pipe = blocks.SpeakerDiarization(c)
        pipe(chunks[:256])                     # first call: handles, staging (not timed), then a fresh run
        pipe.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe.set_timestamp_shift(-fw.padding[0])
        acc = PredictionAccumulator(uri)
        for i in range(0, len(chunks), 256):
            for out in pipe(chunks[i:i + 256]):
                acc.on_next(out)
        preds.append(acc.get_prediction())
        secs.append(time.perf_counter() - t0)
    return preds, secs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=30.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    result = {"card": card()}
    config = make_config(dev)
    x = synth.synth_audio(int(args.minutes * 60 * 16000), seed=2024, num_speakers=5)
    fw = file_windows(x, config)
    sweep = HyperParameterSweep(config)
    sweep.run(x, uri="synth", trials=trials(4))           # warm-up: handles, pinned staging, first-use attributes
    result["chunks"] = fw.num_windows
    result["file_seconds"] = len(x) / 16000
    rows = {}
    for T in (1, 16, 64, 256):
        sweep.run(x, uri="synth", trials=trials(T))
        best = dict(sweep.timing)
        for _ in range(2):
            preds = sweep.run(x, uri="synth", trials=trials(T))
            best = {k: min(best[k], v) for k, v in sweep.timing.items()}
        rows[T] = {"network_s": best["network"], "sweep_device_s": best["sweep"], "assembly_s": best["assembly"],
                   "total_s": best["network"] + best["sweep"] + best["assembly"],
                   "turn_lines": int(sum(p.to_rttm().count("\n") for p in preds))}
        if T == 16:
            want, secs = baseline(config, fw, trial_params(trials(16), config), "synth")
            same = [a.to_rttm() == b.to_rttm() for a, b in zip(preds, want)]
            rows[T]["baseline_sequential_s"] = float(sum(secs))
            rows[T]["baseline_per_run_s"] = float(np.median(secs))
            rows[T]["baseline_equal"] = all(same)
            rows[T]["speedup"] = rows[T]["baseline_sequential_s"] / rows[T]["total_s"]
    result["trials"] = rows
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not rows[16]["baseline_equal"]:
        sys.exit("the sweep's predictions differ from sequential pipeline runs")


if __name__ == "__main__":
    main()
