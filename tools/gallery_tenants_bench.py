"""Measures per-stream galleries at 4 096 streams, one window per stream and tick, and prints one JSON line (and writes it to
--out if given).

Every gallery holds random entries at threshold 0.5, so that no speaker is ever named and every active speaker is searched
at every tick -- the most work a tick can have (as in tools/gallery_bench.py).  The workloads:

    shared     one server whose default gallery has --shared entries
    tenants    one server, --tenants galleries of --tenant-size entries, each given to N / tenants streams with open(gallery=)
    rosters    one server, each stream its own gallery of --roster entries
    split      the tenants workload as --tenants servers of N / tenants streams each (device time summed): one gallery per
               server, what serving tenants apart costs

tick: device_ms per tick from dg_multi_last_step_ms, and host_ms (the tick's wall clock less its device time: pushing,
planning, the annotations) and call_ms (the wall clock of dg_multi_step, the gallery plan included;
tools/multi_stream_config_bench.py) over --ticks ticks after
--warmup, the workloads alternated --rounds times in one process.  kernels: a separate run per workload with
per-kernel event timing (dg_profile_enable): gallery_queries, gallery_nearest and gallery_claim per tick.  The card's name
and power limit are recorded with the numbers.

    python tools/gallery_tenants_bench.py [--streams 4096] [--rounds 3] [--out /tmp/tenants.json]
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

import torch  # noqa: E402

from diart_b200 import _lib, serve  # noqa: E402
from gallery_bench import random_gallery  # noqa: E402
from multi_stream_bench import block, stream_audio  # noqa: E402
from multi_stream_config_bench import run  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402


def workload(name, config, n, galleries):
    """[(server, [open kwargs of each of its streams])] of a workload"""
    if name == "shared":
        return [(serve.MultiStreamDiarization(config, n, 1, gallery=galleries["shared"]), [{}] * n)]
    if name == "tenants":
        per = n // len(galleries["tenants"])
        return [(serve.MultiStreamDiarization(config, n, 1), [dict(gallery=g) for g in galleries["tenants"] for _ in range(per)])]
    if name == "rosters":
        return [(serve.MultiStreamDiarization(config, n, 1), [dict(gallery=g) for g in galleries["rosters"]])]
    if name == "split":
        per = n // len(galleries["tenants"])
        return [(serve.MultiStreamDiarization(config, per, 1, gallery=g), [{}] * per) for g in galleries["tenants"]]
    raise ValueError(name)


def profile(groups, ticks, warmup):
    """per-kernel event timing (ms per tick, summed over the servers) of `ticks` ticks after `warmup`"""
    lib = _lib.lib()
    n = sum(len(kws) for _, kws in groups)
    audios = iter(stream_audio(n, ticks + warmup))
    streams = [[(srv.open(**kw), next(audios)) for kw in kws] for srv, kws in groups]
    buf = C.create_string_buffer(1 << 16)
    for t in range(warmup + ticks):
        if t == warmup:
            lib.dg_profile_report(buf, len(buf))    # drop what the warm-up recorded
            lib.dg_profile_enable(1)
        for srv, ss in zip((g[0] for g in groups), streams):
            for sid, a in ss:
                srv.push(sid, block(a, t))
            srv.step()
    lib.dg_profile_report(buf, len(buf))
    lib.dg_profile_enable(0)
    rep = json.loads(buf.value.decode())
    return {k: round(v["ms"] / ticks, 3) for k, v in rep.items() if k.startswith("gallery") or k == "cluster_sweep"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--shared", type=int, default=10000)
    ap.add_argument("--tenants", type=int, default=64)
    ap.add_argument("--tenant-size", type=int, default=1000)
    ap.add_argument("--roster", type=int, default=16)
    ap.add_argument("--workloads", default="shared,tenants,rosters,split")
    ap.add_argument("--ticks", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gallery_tenants_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    config = make_config(dev)
    D, n = 512, args.streams
    galleries = {"shared": random_gallery(args.shared, D, dev),
                 "tenants": [random_gallery(args.tenant_size, D, dev, seed=1 + i) for i in range(args.tenants)],
                 "rosters": [random_gallery(args.roster, D, dev, seed=10000 + i) for i in range(n)]}
    names = args.workloads.split(",")
    result = {"card": card(), "streams": n, "ticks": args.ticks, "warmup": args.warmup, "rounds": args.rounds,
              "sizes": {"shared": args.shared, "tenants": [args.tenants, args.tenant_size], "roster": args.roster},
              "tick": {k: [] for k in names}, "host_ms": {k: [] for k in names},
              "call_ms": {k: [] for k in names}}
    for _ in range(args.rounds):
        for name in names:
            r = run(workload(name, config, n, galleries), args.ticks, args.warmup)
            result["tick"][name].append(r["device_ms"])
            result["host_ms"][name].append(r["host_ms"])
            result["call_ms"][name].append(r["call_ms"])
            gc.collect()
        print(json.dumps({"device_ms": result["tick"], "host_ms": result["host_ms"]}), flush=True)
    result["spread"] = {k: [min(v), max(v)] for k, v in result["tick"].items()}
    result["host_spread"] = {k: [min(v), max(v)] for k, v in result["host_ms"].items()}
    result["kernels"] = {}
    for name in names:
        result["kernels"][name] = profile(workload(name, config, n, galleries), args.ticks, args.warmup)
        gc.collect()
    print(json.dumps({"kernels": result["kernels"]}), flush=True)
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
