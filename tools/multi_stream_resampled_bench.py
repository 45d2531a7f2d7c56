"""Measures serving N live streams at their own source rates from one MultiStreamDiarization on the GPU, and prints one JSON
line (and writes it to --out if given).

Every tick pushes 0.5 s (one step) of seeded synthetic audio at the stream's rate to every stream and steps once, so each
stream gives one window per tick.  Traffic mixes: all at 16 kHz, all at 44.1 kHz, all at 48 kHz, and a third at each of
16 / 44.1 / 48 kHz; for every N the 16 kHz mix and the resampled mixes alternate (16, 44.1, 16, 48, 16, mixed) on one server
with the three rates declared, so each resampled mix has a 16 kHz run beside it.  Per tick over --ticks ticks after
--warmup (means):

    device_ms     CUDA events on the handle's stream around the tick's device work (dg_multi_last_step_ms)
    resample_ms   the resampling kernels of the tick (profiling tags resample_frames + resample_gather), in a separate run
                  of --ticks ticks with per-kernel events on
    wall_ms       push of every stream's block + step(), host clock

Baseline for N <= --baseline-max (default 64), resampled mixes only: N dedicated pipelines, each __call__ with its one
window per tick, the window resampled by DeviceResample (the reference's live mode with blocks.Resample).  The card's name
and power limit are recorded with the numbers.

    python tools/multi_stream_resampled_bench.py [--streams 64,256,1024,4096] [--out /tmp/multi_stream_resampled.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from diart_b200 import _lib, blocks, serve, synth  # noqa: E402
from diart_b200.core import SlidingWindow, SlidingWindowFeature  # noqa: E402
from diart_b200.operators import DeviceResample  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402

SR = 16000
RATES = (44100, 48000)
MIXES = {"16k": (SR,), "44.1k": (44100,), "48k": (48000,), "mixed": (SR, 44100, 48000)}
ORDER = ["16k", "44.1k", "16k", "48k", "16k", "mixed"]


def stream_audio(rates, ticks):
    """per stream: chunk + (ticks - 1) hop samples at its rate, slices of a few seeded recordings at per-stream offsets"""
    base, out = {}, []
    for i, r in enumerate(rates):
        chunk, hop, _ = serve.source_geometry(r, SR, 5.0, 0.5)
        need = chunk + (ticks - 1) * hop
        if r not in base:
            base[r] = [synth.synth_audio(need + 16 * hop, seed=900 + j, sample_rate=r) for j in range(4)]
        out.append((r, chunk, hop, base[r][i % 4][(i // 4) % 16 * hop:][:need]))
    return out


def block(chunk, hop, a, t):
    return a[:chunk] if t == 0 else a[chunk + (t - 1) * hop:chunk + t * hop]


def profile_tags():
    buf = C.create_string_buffer(1 << 20)
    _lib.lib().dg_profile_report(buf, len(buf))
    return json.loads(buf.value.decode())


def run_server(srv, mix, n, ticks, warmup):
    rates = [MIXES[mix][i % len(MIXES[mix])] for i in range(n)]
    streams = stream_audio(rates, 2 * ticks + warmup)
    sids = [srv.open(sample_rate=r) for r in rates]
    lib = _lib.lib()
    acc = {"wall_ms": 0.0, "device_ms": 0.0}
    rs_ms = 0.0
    for t in range(warmup + 2 * ticks):
        profiled = t >= warmup + ticks
        if t == warmup + ticks:
            lib.dg_profile_enable(1)
        t0 = time.perf_counter()
        for sid, (_, chunk, hop, a) in zip(sids, streams):
            srv.push(sid, block(chunk, hop, a, t))
        out = srv.step()
        t1 = time.perf_counter()
        assert sum(len(v) for v in out.values()) == n
        if t >= warmup and not profiled:
            ms = C.c_float()
            _lib.check(lib.dg_multi_last_step_ms(srv.handle, C.byref(ms)))
            acc["device_ms"] += ms.value
            acc["wall_ms"] += (t1 - t0) * 1e3
    tags = profile_tags()
    lib.dg_profile_enable(0)
    rs_ms = sum(tags.get(k, {}).get("ms", 0.0) for k in ("resample_frames", "resample_gather"))
    for sid in sids:
        srv.close(sid)
    r = {k: round(v / ticks, 3) for k, v in acc.items()}
    r["resample_ms"] = round(rs_ms / ticks, 3)
    r["windows_per_s"] = round(n / (r["wall_ms"] / 1e3), 1)
    return r


def run_baseline(config, mix, n, ticks, warmup):
    rates = [MIXES[mix][i % len(MIXES[mix])] for i in range(n)]
    streams = stream_audio(rates, ticks + warmup)
    dev = config.device
    rs = {r: DeviceResample(r, SR, dev) for r in set(rates) if r != SR}
    pipes = [blocks.SpeakerDiarization(config) for _ in range(n)]
    total = 0.0
    for t in range(warmup + ticks):
        t0 = time.perf_counter()
        for p, (r, chunk, hop, a) in zip(pipes, streams):
            x = torch.from_numpy(np.ascontiguousarray(a[t * hop:t * hop + chunk])).to(dev)
            res = 1 / SR
            if r != SR:
                x = rs[r](x)
                res = (chunk * (1 / r)) / x.shape[0]
            w = SlidingWindowFeature(x.cpu().numpy()[:, None], SlidingWindow(start=t * 0.5, duration=res, step=res))
            p([w])
        if t >= warmup:
            total += time.perf_counter() - t0
    wall = total / ticks * 1e3
    return {"wall_ms": round(wall, 3), "windows_per_s": round(n / (wall / 1e3), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="64,256,1024,4096")
    ap.add_argument("--ticks", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--baseline-max", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_stream_resampled_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    config = make_config(dev)
    result = {"card": card(), "ticks": args.ticks, "warmup": args.warmup, "order": ORDER, "server": {}, "dedicated": {}}
    for n in [int(x) for x in args.streams.split(",")]:
        srv = serve.MultiStreamDiarization(config, max_streams=n, max_windows_per_stream=1, source_sample_rates=RATES)
        runs = {}
        for mix in ORDER:
            runs.setdefault(mix, []).append(run_server(srv, mix, n, args.ticks, args.warmup))
        del srv
        torch.cuda.empty_cache()
        result["server"][n] = runs
        if n <= args.baseline_max:
            result["dedicated"][n] = {mix: run_baseline(config, mix, n, args.ticks, args.warmup) for mix in ("44.1k", "48k")}
        print(json.dumps({"streams": n, "server": runs, "dedicated": result["dedicated"].get(n)}), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
