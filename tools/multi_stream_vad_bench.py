"""Measures serving N live VAD streams from one MultiStreamVoiceActivityDetection on the GPU, against N dedicated
VoiceActivityDetection pipelines called with one window each (the reference's live mode) and against a MultiStreamDiarization
at the same N, and prints one JSON line (and writes it to --out if given).

Every tick pushes 0.5 s (one step) of seeded synthetic audio to every stream and steps once, so each stream gives one window
per tick, as a live stream does.  For N in --streams, after --warmup ticks, per tick over --ticks ticks (means), the phases of
tools/multi_stream_bench.py:

    wall_ms       push of every stream's block + step(), host clock
    push_ms       the pushes (copies into pinned staging)
    call_ms       host clock around the synchronous dg_multi_step library call (device work, launches and host set-up)
    device_ms     CUDA events on the handle's stream around the tick's device work (dg_multi_last_step_ms)
    plan_ms, annotations_ms   host work of step() around the call
    windows_per_s N / wall

The default N go past 4096 up to 65 535, the most a handle takes (max_streams * max_windows_per_stream <= 65 535), to find
the largest N whose tick stays under the 0.5 s step.  For N <= --diarization-max the VAD server and a MultiStreamDiarization
on the same segmentation weights run alternately, --rounds times each, so the difference is what dropping the embedding
network and the clustering saves per tick.  Baseline for N <= --baseline-max: N VoiceActivityDetection pipelines, each
__call__ with its one window per tick.  The card's name and power limit are recorded with the numbers.

    python tools/multi_stream_vad_bench.py [--streams 1,64,256,1024,4096,16384,32768,65535] [--out /tmp/vad_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from diart_b200 import _lib, blocks, serve  # noqa: E402
from diart_b200.core import SlidingWindow, SlidingWindowFeature  # noqa: E402
from multi_stream_bench import run_server, stream_audio  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402

SR, S, HOP = 16000, 80000, 8000


def run_baseline(config, n, ticks, warmup):
    audios = stream_audio(n, ticks + warmup)
    pipes = [blocks.VoiceActivityDetection(config) for _ in range(n)]
    total = 0.0
    for t in range(warmup + ticks):
        t0 = time.perf_counter()
        for p, a in zip(pipes, audios):
            w = SlidingWindowFeature(a[t * HOP:t * HOP + S, None], SlidingWindow(start=t * 0.5, duration=1 / SR, step=1 / SR))
            p([w])
        if t >= warmup:
            total += time.perf_counter() - t0
    wall = total / ticks * 1e3
    return {"wall_ms": round(wall, 3), "windows_per_s": round(n / (wall / 1e3), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,64,256,1024,4096,16384,32768,65535")
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--diarization-max", type=int, default=4096)
    ap.add_argument("--baseline-max", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_stream_vad_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    dia_cfg = make_config(dev)
    vad_cfg = blocks.VoiceActivityDetectionConfig(segmentation=dia_cfg.segmentation, device=dev)
    result = {"card": card(), "ticks": args.ticks, "warmup": args.warmup, "rounds": args.rounds, "step_s": vad_cfg.step,
              "server": {}, "diarization_server": {}, "dedicated": {}}
    for n in [int(x) for x in args.streams.split(",")]:
        vad_runs, dia_runs = [], []
        try:
            for _ in range(args.rounds):
                vad_runs.append(run_server(vad_cfg, n, args.ticks, args.warmup, serve.MultiStreamVoiceActivityDetection))
                gc.collect()             # the handle of the last run frees its rings before the next one allocates
                if n <= args.diarization_max:
                    dia_runs.append(run_server(dia_cfg, n, args.ticks, args.warmup, serve.MultiStreamDiarization))
                    gc.collect()
        except _lib.DiartB200Error as e:   # device or pinned host memory ran out at this N: recorded, the larger N skipped
            result["error"] = {"streams": n, "message": str(e)}
            print(json.dumps(result["error"]), flush=True)
            break
        result["server"][n] = vad_runs
        if dia_runs:
            result["diarization_server"][n] = dia_runs
        if n <= args.baseline_max:
            result["dedicated"][n] = run_baseline(vad_cfg, n, args.ticks, args.warmup)
        print(json.dumps({"streams": n, "server": vad_runs, "diarization_server": dia_runs or None,
                          "dedicated": result["dedicated"].get(n)}), flush=True)
    under = [n for n, runs in result["server"].items() if max(r["wall_ms"] for r in runs) < vad_cfg.step * 1e3]
    result["largest_n_under_step"] = max(under) if under else None
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
