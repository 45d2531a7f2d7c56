"""Measures a dataset sweep over G overlap-aware weightings (DatasetSweep(..., osp=...): one network pass, the embeddings of
every OSP set) against G single-set DatasetSweeps built one after another (one network pass each), on the GPU, and prints one
JSON line (and writes it to --out if given).

Dataset: the 32 seeded files of tools/sweep_dataset_bench.py (about 4.8 h).  OSP sets: G in {1, 4, 16}, a gamma x beta grid
(gamma in {3, 2, 1, 2.5}, beta in {10, 5, 7, 20}; G = 4 takes gamma in {3, 2} x beta in {10, 5}).  For each G:

    construct_s / resident_gb         DatasetSweep(config, files, osp=sets)
    singles_construct_s / _gb         the G single-set sweeps, each at its set's config, built one after another (summed)
    score[T]                          score() of T in {16, 256} trials spread over the sets: host clock of the call and CUDA
                                      events around the launches, against the same trials split over the G single-set sweeps

and the per-set network cost from the profile tags osp, tdnn5 and emb_linear (dg_profile_report over a construction of the
first four files at G = 1 and G = 16: (ms at 16 - ms at 1) / 15).  Every (file, trial) component must be equal bit for bit to
the single-set sweep's (exit status 1 otherwise).  The card's name and power limit are recorded with the numbers.

    python tools/osp_sweep_bench.py [--files 32] [--out /tmp/osp_sweep_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes
import itertools
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
from diart_b200.tune import DatasetSweep, HyperParameterSweep  # noqa: E402
from sweep_bench import card, make_config, trials  # noqa: E402
from sweep_dataset_bench import make_dataset  # noqa: E402

GAMMAS, BETAS = (3, 2, 1, 2.5), (10, 5, 7, 20)
TAGS = ("osp", "pool_weights", "tdnn5", "pool_finalize", "emb_linear", "l2norm")


def grid(G):
    n = {1: 1, 4: 2, 16: 4}[G]
    return [{"gamma": g, "beta": b} for g, b in itertools.product(GAMMAS[:n], BETAS[:n])]


def spread(T, sets):
    """T trials of sweep_bench.trials, trial i at set i mod G"""
    return [dict(t, **sets[i % len(sets)]) for i, t in enumerate(trials(T))]


def profile(config, files, sets):
    lib = _lib.lib()
    lib.dg_profile_report(ctypes.create_string_buffer(1 << 16), 1 << 16)     # drop earlier records
    lib.dg_profile_enable(1)
    try:
        DatasetSweep(config, files, osp=sets[1:])
        buf = ctypes.create_string_buffer(1 << 16)
        lib.dg_profile_report(buf, len(buf))
    finally:
        lib.dg_profile_enable(0)
    rep = json.loads(buf.value.decode())
    return {t: rep.get(t, {"ms": 0.0})["ms"] for t in TAGS}


def timed_score(ds, tr):
    best_call, best_dev = None, None
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        per_file, _ = ds.score(tr)
        call = time.perf_counter() - t0
        best_call = call if best_call is None else min(best_call, call)
        best_dev = ds.timing["score"] if best_dev is None else min(best_dev, ds.timing["score"])
    return per_file, best_call, best_dev


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
    result["audio_hours"] = sum(len(x) for _, x, _ in files) / 16000 / 3600
    HyperParameterSweep(config).score(files[0][1][:60 * 16000], files[0][2], trials(4))    # warm-up
    DatasetSweep(config, files[:2], osp=grid(4)[1:]).score(spread(4, grid(4)))
    rows, equal = {}, True
    for G in (1, 4, 16):
        sets = grid(G)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ds = DatasetSweep(config, files, osp=sets[1:])
        row = {"construct_s": time.perf_counter() - t0, "resident_gb": ds.resident_bytes / 1e9}
        got = {T: timed_score(ds, spread(T, sets)) for T in (16, 256)}
        del ds
        # the G single-set sweeps, one after another, each scoring its share of the trials
        single_s, single_b = 0.0, 0
        want = {T: [np.empty((T, 5)) for _ in files] for T in got}
        split_call, split_dev = {T: 0.0 for T in got}, {T: 0.0 for T in got}
        for g, s in enumerate(sets):
            cfg = make_config(dev, **s)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            one = DatasetSweep(cfg, files)
            single_s += time.perf_counter() - t0
            single_b += one.resident_bytes
            for T in got:
                pos = list(range(g, T, G))
                per_file, call, dev_s = timed_score(one, [trials(T)[i] for i in pos])
                split_call[T] += call
                split_dev[T] += dev_s
                for f, comp in enumerate(per_file):
                    want[T][f][pos] = comp.as_array()
            del one
        row.update({"singles_construct_s": single_s, "singles_resident_gb": single_b / 1e9})
        row["score"] = {}
        for T, (per_file, call, dev_s) in got.items():
            same = all(np.array_equal(p.as_array(), w) for p, w in zip(per_file, want[T]))
            equal &= same
            row["score"][T] = {"call_s": call, "device_s": dev_s, "split_call_s": split_call[T],
                               "split_device_s": split_dev[T], "components_equal": same}
        rows[G] = row
        print(json.dumps({G: row}), file=sys.stderr)
    result["sets"] = rows
    p1, p16 = profile(config, files[:4], grid(1)), profile(config, files[:4], grid(16))
    result["profile_4_files_ms"] = {"G1": p1, "G16": p16,
                                    "per_extra_set": {t: (p16[t] - p1[t]) / 15 for t in TAGS}}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
