"""Measures serving N live streams from one MultiStreamDiarization on the GPU, and N dedicated SpeakerDiarization pipelines
called with one window each as the baseline (the reference's live mode, StreamingInference(batch_size=1) per stream), and
prints one JSON line (and writes it to --out if given).

Every tick pushes 0.5 s (one step) of seeded synthetic audio to every stream and steps once, so each stream gives one window
per tick, as a live stream does.  For N in --streams (default 1, 64, 256, 1024, 4096), after --warmup ticks, per tick over
--ticks ticks (means):

    wall_ms       push of every stream's block + step(), host clock
    push_ms       the pushes (copies into pinned staging)
    call_ms       host clock around the synchronous dg_multi_step library call (device work, launches and host set-up)
    device_ms     CUDA events on the handle's stream around the tick's device work: one upload, scatter / gather,
                  networks, clustering, post-path, one download (dg_multi_last_step_ms)
    plan_ms, annotations_ms   host work of step() around the call
    windows_per_s N / wall

and the largest N whose tick stays under the 0.5 s step.  Baseline for N <= --baseline-max (default 64): N pipelines, each
__call__ with its one window per tick.  The card's name and power limit are recorded with the numbers.

    python tools/multi_stream_bench.py [--streams 1,64,256,1024,4096] [--out /tmp/multi_stream_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import functools
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from diart_b200 import _lib, blocks, serve, synth  # noqa: E402
from diart_b200.core import SlidingWindow, SlidingWindowFeature  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402

SR, S, HOP = 16000, 80000, 8000


@functools.lru_cache(maxsize=4)
def recordings(need):
    """the seeded recordings the streams are cut from (synthesised once per length: seconds each)"""
    return [synth.synth_audio(need + 64 * HOP, seed=900 + i) for i in range(8)]


def stream_audio(n_streams, ticks):
    """per stream: S + (ticks - 1) HOP samples, slices of a few seeded recordings at per-stream offsets"""
    need = S + (ticks - 1) * HOP
    base = recordings(need)
    return [base[i % 8][(i // 8) % 64 * HOP:][:need] for i in range(n_streams)]


def block(a, t):
    return a[:S] if t == 0 else a[S + (t - 1) * HOP:S + t * HOP]


def timed_step(srv, phases):
    """srv.step() with the host clock around its phases (the same code path, instrumented); any multi-stream server"""
    t0 = time.perf_counter()
    plan_rows, annotations = serve.plan_rows, srv._annotations
    marks = {}

    def plan(*a, **k):
        r = plan_rows(*a, **k)
        marks["plan"] = time.perf_counter()
        return r

    def ann(*a, **k):
        marks["ann0"] = time.perf_counter()
        return annotations(*a, **k)

    serve.plan_rows, srv._annotations = plan, ann
    try:
        out = srv.step()
    finally:
        serve.plan_rows = plan_rows
        del srv._annotations
    t1 = time.perf_counter()
    phases["plan_ms"] += (marks["plan"] - t0) * 1e3
    phases["call_ms"] += (marks["ann0"] - marks["plan"]) * 1e3
    phases["annotations_ms"] += (t1 - marks["ann0"]) * 1e3
    ms = C.c_float()
    _lib.check(_lib.lib().dg_multi_last_step_ms(srv.handle, C.byref(ms)))
    phases["device_ms"] += ms.value
    return out


def run_server(config, n, ticks, warmup, server=serve.MultiStreamDiarization):
    audios = stream_audio(n, ticks + warmup)
    srv = server(config, max_streams=n, max_windows_per_stream=1)
    sids = [srv.open() for _ in range(n)]
    phases = {k: 0.0 for k in ("wall_ms", "push_ms", "plan_ms", "call_ms", "device_ms", "annotations_ms")}
    for t in range(warmup + ticks):
        if t == warmup:
            phases = {k: 0.0 for k in phases}
        t0 = time.perf_counter()
        for sid, a in zip(sids, audios):
            srv.push(sid, block(a, t))
        t1 = time.perf_counter()
        out = timed_step(srv, phases)
        t2 = time.perf_counter()
        assert sum(len(v) for v in out.values()) == n
        phases["push_ms"] += (t1 - t0) * 1e3
        phases["wall_ms"] += (t2 - t0) * 1e3
    r = {k: round(v / ticks, 3) for k, v in phases.items()}
    r["windows_per_s"] = round(n / (r["wall_ms"] / 1e3), 1)
    return r


def run_baseline(config, n, ticks, warmup):
    audios = stream_audio(n, ticks + warmup)
    pipes = [blocks.SpeakerDiarization(config) for _ in range(n)]
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
    ap.add_argument("--streams", default="1,64,256,1024,4096")
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--baseline-max", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_stream_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    config = make_config(dev)
    result = {"card": card(), "ticks": args.ticks, "warmup": args.warmup, "step_s": config.step, "server": {}, "dedicated": {}}
    for n in [int(x) for x in args.streams.split(",")]:
        result["server"][n] = run_server(config, n, args.ticks, args.warmup)
        if n <= args.baseline_max:
            result["dedicated"][n] = run_baseline(config, n, args.ticks, args.warmup)
        print(json.dumps({"streams": n, "server": result["server"][n], "dedicated": result["dedicated"].get(n)}), flush=True)
    under = [n for n, r in result["server"].items() if r["wall_ms"] < config.step * 1e3]
    result["largest_n_under_step"] = max(under) if under else None
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
