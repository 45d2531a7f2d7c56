"""Measures what gallery naming costs, and prints one JSON line (and writes it to --out if given).

    tick       MultiStreamDiarization with N streams (--streams), one window per stream and tick: per tick over --ticks ticks
               after --warmup, device_ms from dg_multi_last_step_ms and the other phases of tools/multi_stream_config_bench.py.
               `none`: no gallery; `G=<n>`: a gallery of n random entries (--galleries) at threshold 0.5, so that no speaker
               is ever named and every active speaker is compared at every tick -- the most work a tick can have at that
               gallery size.  All variants alternated --rounds times in one process.
    kernels    a separate run with per-kernel event timing (dg_profile_enable): gallery_queries, gallery_nearest and
               gallery_claim per tick, at the largest stream count and every gallery size, with the tick's query count.
    query      dg_gallery_query alone at Q = --q queries (groups of 4), G = --g entries, D = 512: device time from CUDA events
               over --reps calls after a warm-up, and the float64 rate 2 Q G D / time against the H100 SXM data sheet's 67
               TFLOP/s FP64 tensor-core rate.

The card's name and power limit are recorded with the numbers.

    python tools/gallery_bench.py [--streams 1024,4096] [--galleries 1000,10000,100000] [--out /tmp/gallery.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from diart_b200 import _lib, serve  # noqa: E402
from diart_b200.speakers import KnownSpeakers, SpeakerGallery  # noqa: E402
from multi_stream_bench import block, stream_audio  # noqa: E402
from multi_stream_config_bench import run  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402

FP64_TC_TFLOPS = 67.0     # NVIDIA H100 SXM data sheet, dense FP64 tensor core


def random_gallery(G, D, dev, seed=0):
    rng = np.random.default_rng(seed)
    return SpeakerGallery(KnownSpeakers([f"e{i}" for i in range(G)], rng.standard_normal((G, D))), 0.5, dev)


def profile(config, n, gallery, ticks, warmup):
    """per-kernel event timing of `ticks` ticks after `warmup`, one window per stream and tick"""
    lib = _lib.lib()
    server = serve.MultiStreamDiarization(config, n, 1, gallery=gallery)
    audios = stream_audio(n, ticks + warmup)
    sids = [server.open() for _ in range(n)]
    buf = C.create_string_buffer(1 << 16)
    for t in range(warmup + ticks):
        if t == warmup:
            lib.dg_profile_report(buf, len(buf))    # drop what the warm-up recorded
            lib.dg_profile_enable(1)
        for sid, a in zip(sids, audios):
            server.push(sid, block(a, t))
        server.step()
    lib.dg_profile_report(buf, len(buf))
    lib.dg_profile_enable(0)
    rep = json.loads(buf.value.decode())
    out = {k: round(v["ms"] / ticks, 3) for k, v in rep.items() if k.startswith("gallery") or k == "cluster_sweep"}
    out["active_speakers_at_end"] = sum(len(server.speakers(s)) for s in sids)
    return out


def bench_query(dev, Q, G, D, reps):
    gal = random_gallery(G, D, dev, seed=1)
    rng = np.random.default_rng(2)
    x = torch.from_numpy(rng.standard_normal((Q, D))).to(dev)
    group = torch.from_numpy(np.repeat(np.arange(Q // 4), 4).astype(np.int32)).to(dev)
    claimed = torch.full((Q // 4, 32), -1, dtype=torch.int32, device=dev)
    entry = torch.empty(Q, dtype=torch.int32, device=dev)
    dist = torch.empty(Q, dtype=torch.float64, device=dev)
    lib = _lib.lib()
    st = _lib.stream_ptr(dev)

    def call():
        _lib.check(lib.dg_gallery_query(gal.handle, x.data_ptr(), Q, group.data_ptr(), claimed.data_ptr(), gal.threshold,
                                        entry.data_ptr(), dist.data_ptr(), st))

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    ms = float(np.median(times))
    flop = 2.0 * Q * G * D
    return {"Q": Q, "G": G, "D": D, "ms_median": round(ms, 3), "ms_min": round(min(times), 3),
            "tflops": round(flop / (ms * 1e-3) / 1e12, 2), "share_of_fp64_tc_datasheet": round(flop / (ms * 1e-3) / 1e12 /
                                                                                               FP64_TC_TFLOPS, 3),
            "note": "includes the call's read-back of the groups (one small copy and a synchronise)"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1024,4096")
    ap.add_argument("--galleries", default="1000,10000,100000")
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--q", type=int, default=16384)
    ap.add_argument("--g", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gallery_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    config = make_config(dev)
    D = 512
    sizes = [int(x) for x in args.galleries.split(",")]
    galleries = {G: random_gallery(G, D, dev) for G in sizes}
    result = {"card": card(), "ticks": args.ticks, "warmup": args.warmup, "rounds": args.rounds, "tick": {}}
    for n in [int(x) for x in args.streams.split(",")]:
        rows = {"none": []}
        rows.update({f"G={G}": [] for G in sizes})
        for _ in range(args.rounds):
            for key in rows:
                gal = None if key == "none" else galleries[int(key[2:])]
                rows[key].append(run([(serve.MultiStreamDiarization(config, n, 1, gallery=gal), [{}] * n)], args.ticks,
                                     args.warmup))
                gc.collect()
        result["tick"][n] = {k: [r["device_ms"] for r in v] for k, v in rows.items()}
        print(json.dumps({"streams": n, "device_ms": result["tick"][n]}), flush=True)
    n = max(int(x) for x in args.streams.split(","))
    result["kernels"] = {"streams": n}
    for G in sizes:
        result["kernels"][f"G={G}"] = profile(config, n, galleries[G], args.ticks, args.warmup)
        gc.collect()
    print(json.dumps({"kernels": result["kernels"]}), flush=True)
    result["query"] = bench_query(dev, args.q, args.g, D, args.reps)
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
