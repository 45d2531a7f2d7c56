"""Measures what a scoring protocol costs a dataset sweep on the GPU: DatasetSweep.score under the default metric, under
DiarizationErrorRate(collar=0.25, skip_overlap=True), and under that metric with a uem per file, and prints one JSON line
(and writes it to --out if given).

Dataset: the seeded synthetic files of tools/sweep_dataset_bench.py (--files, default 32, about 4.8 h).  The uem of a file
of duration D leaves out 10 % of it in three pieces of D / 30 at 0.2 D, 0.5 D and 0.8 D.  For T in {1, 16, 256} trials and
each metric:

    call_s          host clock of score() (best of 3)
    score_device_s  CUDA events around the scoring launches (best of 3)
    der_score_ms    the der_score kernel's CUDA-event time from dg_profile_report, in a profiled call of its own
    regions_pack_s  host time of the first call under the metric: scored regions and cropped references of every file
                    (later calls reuse them)

The default metric's components must equal those of score() without a metric, bit for bit (exit status 1 otherwise).  The
card's name and power limit are recorded with the numbers.

    python tools/sweep_protocol_bench.py [--files 32] [--out /tmp/sweep_protocol_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from diart_b200 import _lib  # noqa: E402
from diart_b200.tune import DatasetSweep, DiarizationErrorRate, HyperParameterSweep  # noqa: E402
from sweep_bench import card, make_config, trials  # noqa: E402
from sweep_dataset_bench import SR, make_dataset  # noqa: E402


def file_uem(duration: float):
    """the file without three pieces of duration / 30 at 0.2, 0.5 and 0.8 of it"""
    g = duration / 30
    cuts = [0.2 * duration, 0.5 * duration, 0.8 * duration]
    starts, ends = [0.0] + [c + g for c in cuts], cuts + [duration]
    return list(zip(starts, ends))


def der_score_ms(call) -> float:
    lib = _lib.lib()
    lib.dg_profile_report(ctypes.create_string_buffer(1 << 16), 1 << 16)     # drop earlier records
    lib.dg_profile_enable(1)
    try:
        call()
        buf = ctypes.create_string_buffer(1 << 16)
        lib.dg_profile_report(buf, len(buf))
    finally:
        lib.dg_profile_enable(0)
    return json.loads(buf.value.decode())["der_score"]["ms"]


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
    result["audio_hours"] = sum(len(x) for _, x, _ in files) / SR / 3600
    sweep = HyperParameterSweep(config)
    plain = DatasetSweep(config, files, sweep=sweep)
    cut = DatasetSweep(config, files, sweep=sweep, uems=[file_uem(len(x) / SR) for _, x, _ in files])
    protocols = {"default": (plain, None), "collar0.25_skip": (plain, DiarizationErrorRate(0.25, True)),
                 "collar0.25_skip_uem": (cut, DiarizationErrorRate(0.25, True))}
    pack = {}
    for name, (ds, metric) in protocols.items():                    # warm-up; the first call packs the regions
        ds.score(trials(4), metric)
        pack[name] = ds.regions_seconds
    result["regions_pack_s"] = pack
    rows, equal = {}, True
    for T in (1, 16, 256):
        tr = trials(T)
        want, _ = plain.score(tr)
        row = {}
        for name, (ds, metric) in protocols.items():
            best_call = best_dev = None
            for _ in range(3):
                t0 = time.perf_counter()
                got, total = ds.score(tr, metric)
                call = time.perf_counter() - t0
                best_call = call if best_call is None else min(best_call, call)
                best_dev = ds.timing["score"] if best_dev is None else min(best_dev, ds.timing["score"])
            kernel = min(der_score_ms(lambda: ds.score(tr, metric)) for _ in range(2))
            row[name] = {"call_s": best_call, "score_device_s": best_dev, "der_score_ms": kernel,
                         "best_der": float(total.der.min())}
            if name == "default":
                same = all(np.array_equal(g.as_array(), w.as_array()) for g, w in zip(got, want))
                row[name]["equals_no_metric"] = same
                equal &= same
        rows[T] = row
    result["trials"] = rows
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not equal:
        sys.exit("the default metric's components differ from score() without a metric")


if __name__ == "__main__":
    main()
