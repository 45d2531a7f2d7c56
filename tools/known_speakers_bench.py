"""Measures what known speakers cost, and prints one JSON line (and writes it to --out if given).

    enroll     diart_b200.speakers.enroll over --clips one-speaker clips of 10 to 30 s (slices of seeded synthetic
               recordings): the DatasetSweep construction (one network pass over every clip) and the sweep (one
               clustering launch, the predictions, the dominant speakers and the gather of their centroids), host clock
               around work that ends in a device synchronise.  Against it, each of the first --baseline-clips clips enrolled
               through its own SpeakerDiarization (fused steps of 32 windows, then speakers()): seconds per clip, and that
               times --clips.  The per-clip run does not even build the clip's prediction, so it is a lower bound of what
               enrolling clip by clip costs.
    tick       MultiStreamDiarization with N streams (--streams), one window per stream and tick: per tick over --ticks ticks
               after --warmup, the phases of tools/multi_stream_config_bench.py, device_ms from dg_multi_last_step_ms.
               `seeded`: every stream opened with 4 known speakers; `plain`: none.  Alternated --rounds times in one
               process.
    open       host seconds of --opens seeded opens (4 known speakers each) and of as many plain ones on a fresh server,
               alternated --rounds times.

The card's name and power limit are recorded with the numbers.

    python tools/known_speakers_bench.py [--clips 1000] [--streams 1024,4096] [--out /tmp/known_speakers.json]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from diart_b200 import blocks, serve, synth  # noqa: E402
from diart_b200.speakers import KnownSpeakers, enroll  # noqa: E402
from diart_b200.tune import file_windows  # noqa: E402
from multi_stream_config_bench import run  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402

SR = 16000


def make_clips(n, seed=0):
    """n one-speaker clips of 10 to 30 s: slices of 8 seeded one-speaker recordings of 125 s"""
    rng = np.random.default_rng(seed)
    base = [synth.synth_audio(125 * SR, seed=5000 + i, num_speakers=1) for i in range(8)]
    clips = []
    for i in range(n):
        length = int(rng.uniform(10, 30) * SR)
        start = int(rng.integers(0, len(base[i % 8]) - length))
        clips.append((f"clip{i}", np.ascontiguousarray(base[i % 8][start:start + length])))
    return clips


def enroll_alone(config, wav, batch=32):
    """one clip through its own SpeakerDiarization: every window in fused steps of ``batch``, then its state"""
    pipe = blocks.SpeakerDiarization(config)
    fw = file_windows(wav, config)
    for i in range(0, fw.num_windows, batch):
        x = np.stack([fw.window(j) for j in range(i, min(i + batch, fw.num_windows))])
        pipe.device_step(torch.from_numpy(x).to(config.device))
    return pipe.speakers()


def bench_enroll(config, n_clips, n_baseline):
    clips = make_clips(n_clips)
    enroll(config, clips[:8])                                   # warm-up: modules, workspaces
    torch.cuda.synchronize()
    timing = {}
    known = enroll(config, clips, timing)
    torch.cuda.synchronize()
    enroll_alone(config, clips[0][1])                           # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _, wav in clips[:n_baseline]:
        enroll_alone(config, wav)
    torch.cuda.synchronize()
    per_clip = (time.perf_counter() - t0) / n_baseline
    audio_s = sum(len(w) for _, w in clips) / SR
    return known, {"clips": n_clips, "audio_hours": round(audio_s / 3600, 3),
                   "construct_s": round(timing["construct"], 3), "sweep_s": round(timing["sweep"], 3),
                   "total_s": round(timing["construct"] + timing["sweep"], 3),
                   "alone_per_clip_s": round(per_clip, 4), "alone_clips_timed": n_baseline,
                   "alone_total_s_scaled": round(per_clip * n_clips, 2)}


def bench_open(config, known, n, rounds):
    out = {"seeded_s": [], "plain_s": []}
    for _ in range(rounds):
        for key, kw in (("seeded_s", dict(speakers=known)), ("plain_s", {})):
            server = serve.MultiStreamDiarization(config, n, 1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n):
                server.open(**kw)
            out[key].append(round(time.perf_counter() - t0, 4))
            del server
            gc.collect()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1000)
    ap.add_argument("--baseline-clips", type=int, default=100)
    ap.add_argument("--streams", default="1024,4096")
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--opens", type=int, default=4096)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("known_speakers_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    config = make_config(dev)
    result = {"card": card(), "ticks": args.ticks, "warmup": args.warmup, "rounds": args.rounds}
    enrolled, result["enroll"] = bench_enroll(config, args.clips, min(args.baseline_clips, args.clips))
    print(json.dumps({"enroll": result["enroll"]}), flush=True)
    known = KnownSpeakers(["alice", "bob", "carol", "dan"], enrolled.centroids[:4])
    result["tick"] = {}
    for n in [int(x) for x in args.streams.split(",")]:
        rows = {"seeded": [], "plain": []}
        for _ in range(args.rounds):
            for key, kw in (("seeded", dict(speakers=known)), ("plain", {})):
                rows[key].append(run([(serve.MultiStreamDiarization(config, n, 1), [kw] * n)], args.ticks, args.warmup))
                gc.collect()
        result["tick"][n] = rows
        print(json.dumps({"streams": n, **rows}), flush=True)
    result["open"] = {"opens": args.opens, **bench_open(config, known, args.opens, args.rounds)}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
