"""Measures what serving every live stream at its own latency and thresholds costs a MultiStreamDiarization tick, and prints
one JSON line (and writes it to --out if given).

Every tick pushes 0.5 s (one step) of seeded synthetic audio to every stream and steps once, so each stream gives one window
per tick.  For N in --streams, after --warmup ticks, per tick over --ticks ticks (means), three ways of serving N streams:

    defaults   one server, every stream at the configuration's values (latency 0.5 s, tau_active 0.6, rho_update 0.3,
               delta_new 1), as a server without per-stream values serves them
    mixed      one server with max_latency 5 s, the streams spread round robin over the reference README's four tuned rows
               (tau_active, rho_update, delta_new) x latencies 0.5, 1, 2 and 5 s: 16 configurations
    split      the mixed streams served by one server per configuration (16 servers, one tick each), device times summed

with the phases of tools/multi_stream_bench.py per tick (summed over the servers of `split`):

    wall_ms       pushes of every stream's block + step() of every server, host clock
    host_ms       wall_ms - device_ms: what the host adds to the device work
    plan_ms, call_ms, annotations_ms   host work of step() before, around and after the dg_multi_step call
    device_ms     CUDA events on the handle's stream around the tick's device work (dg_multi_last_step_ms)

`defaults` and `mixed` run alternately, --rounds times each, in one process; `split` runs once per N after them.  The card's
name and power limit are recorded with the numbers.

    python tools/multi_stream_config_bench.py [--streams 64,256,1024,4096] [--out /tmp/config_bench.json]
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

from diart_b200 import blocks, serve  # noqa: E402
from multi_stream_bench import block, stream_audio, timed_step  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402

# tau_active, rho_update, delta_new of the reference README's table "To obtain the best results" (DIHARD III, AMI,
# VoxConverse, DIHARD II)
README_ROWS = [(0.555, 0.422, 1.517), (0.507, 0.006, 1.057), (0.576, 0.915, 0.648), (0.619, 0.326, 0.997)]
LATENCIES = (0.5, 1.0, 2.0, 5.0)
CONFIGS = [dict(latency=lat, tau_active=t, rho_update=r, delta_new=d) for (t, r, d) in README_ROWS for lat in LATENCIES]
PHASES = ("wall_ms", "push_ms", "plan_ms", "call_ms", "device_ms", "annotations_ms")


def run(groups, ticks, warmup):
    """groups: [(server, [open kwargs of each of its streams])], stepped one after the other every tick -> per tick means"""
    n = sum(len(kws) for _, kws in groups)
    audios = iter(stream_audio(n, ticks + warmup))
    streams = [[(srv.open(**kw), next(audios)) for kw in kws] for srv, kws in groups]
    phases = {k: 0.0 for k in PHASES}
    for t in range(warmup + ticks):
        if t == warmup:
            phases = {k: 0.0 for k in PHASES}
        t0 = time.perf_counter()
        got = 0
        for (srv, _), ss in zip(groups, streams):
            t1 = time.perf_counter()
            for sid, a in ss:
                srv.push(sid, block(a, t))
            phases["push_ms"] += (time.perf_counter() - t1) * 1e3
            got += sum(len(v) for v in timed_step(srv, phases).values())
        phases["wall_ms"] += (time.perf_counter() - t0) * 1e3
        assert got == n
    r = {k: round(v / ticks, 3) for k, v in phases.items()}
    r["host_ms"] = round(r["wall_ms"] - r["device_ms"], 3)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="64,256,1024,4096")
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_stream_config_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    config = make_config(dev)
    result = {"card": card(), "ticks": args.ticks, "warmup": args.warmup, "rounds": args.rounds, "step_s": config.step,
              "configurations": len(CONFIGS), "defaults": {}, "mixed": {}, "split": {}}
    for n in [int(x) for x in args.streams.split(",")]:
        kws = [CONFIGS[i % len(CONFIGS)] for i in range(n)]
        defaults, mixed = [], []
        for _ in range(args.rounds):
            defaults.append(run([(serve.MultiStreamDiarization(config, n, 1), [{}] * n)], args.ticks, args.warmup))
            gc.collect()             # the handle of the last run frees its rings before the next one allocates
            mixed.append(run([(serve.MultiStreamDiarization(config, n, 1, max_latency=5.0), kws)], args.ticks, args.warmup))
            gc.collect()
        groups = []
        for c in CONFIGS:
            members = [kw for kw in kws if kw is c]
            if members:
                own = blocks.SpeakerDiarizationConfig(segmentation=config.segmentation, embedding=config.embedding,
                                                      device=dev, **c)
                groups.append((serve.MultiStreamDiarization(own, len(members), 1), [{}] * len(members)))
        split = run(groups, args.ticks, args.warmup)
        split["servers"] = len(groups)
        del groups
        gc.collect()
        result["defaults"][n], result["mixed"][n], result["split"][n] = defaults, mixed, split
        print(json.dumps({"streams": n, "defaults": defaults, "mixed": mixed, "split": split}), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
