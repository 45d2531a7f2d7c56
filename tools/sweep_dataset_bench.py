"""Measures scoring a dataset of files (DatasetSweep) against scoring it file by file (HyperParameterSweep.score per file,
summed: what HyperParameterSweep.score_files did before the dataset sweep) on the GPU, and prints one JSON line (and writes
it to --out if given).

Dataset: seeded and synthetic, --files files (default 32) with lengths drawn uniformly from 1 to 15 minutes (about 4 h in
all), each a slice of one synthetic 16-minute recording at a seeded offset (generating 4 h of distinct synthetic speech
would take minutes of CPU time per run), each with a seeded 3-6-speaker reference.  For T in {1, 16, 256} trials:

    per_file   HyperParameterSweep.score of every file, summed (network pass + clustering + scoring per file)
    dataset    DatasetSweep.score on the resident network outputs: host clock of the call and CUDA events around the launches

and once: the DatasetSweep construction (the network pass of all files).  The per-file components of the two legs must be
equal bit for bit (exit status 1 otherwise).  The card's name and power limit are recorded with the numbers.

    python tools/sweep_dataset_bench.py [--files 32] [--out /tmp/sweep_dataset_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from diart_b200 import synth  # noqa: E402
from diart_b200.tune import DatasetSweep, HyperParameterSweep  # noqa: E402
from sweep_bench import card, make_config, trials  # noqa: E402
from sweep_score_bench import synth_reference  # noqa: E402

SR = 16000


def make_dataset(n_files, seed=31):
    rng = np.random.default_rng(seed)
    base = synth.synth_audio(16 * 60 * SR, seed=seed, num_speakers=5)
    files = []
    for i in range(n_files):
        n = int(rng.uniform(1.0, 15.0) * 60 * SR)
        a = int(rng.integers(0, len(base) - n + 1))
        x = np.ascontiguousarray(base[a:a + n])
        ref = synth_reference(seed * 100 + i, int(rng.integers(3, 7)), n / SR)
        files.append((f"file{i:02d}", x, ref))
    return files


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
    sweep.score(files[0][1][:60 * SR], files[0][2], trials(4))     # warm-up: handles, staging, first-use attributes
    t0 = time.perf_counter()
    ds = DatasetSweep(config, files)
    result["dataset_construct_s"] = time.perf_counter() - t0
    result["dataset_chunks"] = ds.num_chunks
    result["resident_gb"] = ds.resident_bytes / 1e9
    ds.score(trials(4))                                              # warm-up of the dataset-sized buffers
    rows, equal = {}, True
    for T in (1, 16, 256):
        tr = trials(T)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        want = [sweep.score(x, ref, tr).as_array() for _, x, ref in files]
        per_file_s = time.perf_counter() - t0
        best_call, best_dev = None, None
        for _ in range(3):
            t0 = time.perf_counter()
            got, total = ds.score(tr)
            call = time.perf_counter() - t0
            best_call = call if best_call is None else min(best_call, call)
            best_dev = ds.timing["score"] if best_dev is None else min(best_dev, ds.timing["score"])
        same = all(np.array_equal(g.as_array(), w) for g, w in zip(got, want))
        equal &= same
        rows[T] = {"per_file_s": per_file_s, "dataset_score_call_s": best_call, "dataset_score_device_s": best_dev,
                   "speedup_call": per_file_s / best_call, "components_equal": same, "best_der": float(total.der.min())}
    result["trials"] = rows
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not equal:
        sys.exit("the dataset sweep's components differ from the per-file sweep's")


if __name__ == "__main__":
    main()
