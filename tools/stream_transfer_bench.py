"""Measures moving live streams (MultiStreamDiarization.export / restore) at 1, 256 and 4 096 streams at latency 5 s
(max_windows_per_stream 4, the other values the defaults) and prints one JSON line (and writes it to --out if given).

Every stream pushes its first window and then one hop per tick for --fill ticks (10: its aggregation history holds the
latency / step - 1 = 9 chunks it can), then one more hop that stays staged.  Then, per size:

    warm-up    one export(all, close=False) and restore of the same size, untimed: the staging buffers of both servers
               reach their size (their first growth synchronises the device)
    wall       export(all, close=False) and restore(states) into a second server on the same models, host wall clock,
               profiler off
    kernels    the same two calls again with per-launch event timing (dg_profile_enable): slot_transfer_export /
               slot_transfer_import, and the pinned copies slot_transfer_d2h / slot_transfer_h2d; host_ms = wall - kernel
               - copy (host packing, Python objects)
    bytes      packed bytes per stream
    tick       device time per tick (dg_multi_last_step_ms) of the original and the restored server, --ticks ticks each,
               alternated, every stream pushing one hop per tick

The card's name and power limit are recorded with the numbers.

    python tools/stream_transfer_bench.py [--sizes 1,256,4096] [--out /tmp/transfer.json]
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

from diart_b200 import _lib, serve  # noqa: E402
from multi_stream_bench import block, stream_audio  # noqa: E402
from sweep_bench import card, make_config  # noqa: E402


def kernel_ms(report: dict, name: str) -> float:
    return float(report.get(name, {}).get("ms", 0.0))


def profiled(fn):
    """fn() with per-kernel event timing -> (result, wall ms, {kernel: {count, ms}})"""
    lib = _lib.lib()
    lib.dg_profile_enable(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    wall = (time.perf_counter() - t0) * 1e3
    cbuf = C.create_string_buffer(1 << 16)
    lib.dg_profile_report(cbuf, len(cbuf))
    lib.dg_profile_enable(0)
    return out, wall, json.loads(cbuf.value.decode() or "{}")


def measure(config, n, fill, ticks):
    audio = stream_audio(n, fill + ticks + 2)
    a = serve.MultiStreamDiarization(config, n)
    sids = [a.open() for _ in range(n)]
    for t in range(fill):
        for s in sids:
            a.push(s, block(audio[s], t))
        a.step()
    for s in sids:   # staged, not ticked
        a.push(s, block(audio[s], fill))
    b = serve.MultiStreamDiarization(config, n)

    def move():
        states = a.export(sids, close=False)
        return states, b.restore(states)

    def clear(ids):
        for s in ids:
            b.close(s)

    clear(move()[1])   # warm-up at the measured size
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    states = a.export(sids, close=False)
    t1 = time.perf_counter()
    new = b.restore(states)
    t2 = time.perf_counter()
    clear(new)
    exp_ms, imp_ms = (t1 - t0) * 1e3, (t2 - t1) * 1e3
    states, _, rep_exp = profiled(lambda: a.export(sids, close=False))
    new, _, rep_imp = profiled(lambda: b.restore(states))
    k_exp, c_exp = kernel_ms(rep_exp, "slot_transfer_export"), kernel_ms(rep_exp, "slot_transfer_d2h")
    k_imp, c_imp = kernel_ms(rep_imp, "slot_transfer_import"), kernel_ms(rep_imp, "slot_transfer_h2d")
    res = {"streams": n, "bytes_per_stream": float(np.mean([s.nbytes for s in states])),
           "export": {"wall_ms": exp_ms, "kernel_ms": k_exp, "copy_ms": c_exp, "host_ms": exp_ms - k_exp - c_exp},
           "restore": {"wall_ms": imp_ms, "kernel_ms": k_imp, "copy_ms": c_imp, "host_ms": imp_ms - k_imp - c_imp}}
    dev = {"original": [], "restored": []}
    ms = C.c_float()
    for t in range(ticks):
        for name, srv, ids in (("original", a, sids), ("restored", b, new)):
            for k, s in enumerate(ids):
                srv.push(s, block(audio[sids[k]], fill + 1 + t))
            srv.step()
            _lib.check(_lib.lib().dg_multi_last_step_ms(srv.handle, C.byref(ms)))
            dev[name].append(ms.value)
    res["tick_device_ms"] = {k: {"median": float(np.median(v)), "min": float(np.min(v))} for k, v in dev.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,256,4096")
    ap.add_argument("--fill", type=int, default=10)
    ap.add_argument("--ticks", type=int, default=6)
    ap.add_argument("--out")
    args = ap.parse_args()
    _lib.require_cuda(torch.device("cuda", 0))
    config = make_config(torch.device("cuda", 0), latency=5.0)
    out = {"card": card(), "runs": []}
    for n in [int(x) for x in args.sizes.split(",")]:
        out["runs"].append(measure(config, n, args.fill, args.ticks))
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
