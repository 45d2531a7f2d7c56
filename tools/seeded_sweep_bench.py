"""Measures seeded dataset sweeps and identification error scoring on the GPU, and prints one JSON line (and writes it to
--out if given).

Dataset: the --files files of tools/sweep_dataset_bench.py (default 32, about 4 h).  Gallery: 4 speakers enrolled with
diart_b200.speakers.enroll from one-speaker clips of tools/known_speakers_bench.py; every file is seeded with all 4.  Three
cases over the same resident network outputs, alternated --rounds times in one process, each at T in {1, 16, 256} trials:

    unseeded_der   DatasetSweep(files).score(trials)
    seeded_der     DatasetSweep(files, speakers=gallery).score(trials)
    seeded_ier     the same with metric=IdentificationErrorRate()

score_device_s is the device time of the scoring launches (CUDA events around them, ds.timing["score"]), the best of the
rounds.  Then, in profiled calls of their own at 256 trials, the CUDA-event times of the profile tags sweep_seed and
der_score (dg_profile_report).  The card's name and power limit are recorded with the numbers.

    python tools/seeded_sweep_bench.py [--files 32] [--rounds 3] [--out /tmp/seeded_sweep_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from diart_b200 import _lib  # noqa: E402
from diart_b200.speakers import KnownSpeakers, enroll  # noqa: E402
from diart_b200.tune import DatasetSweep, HyperParameterSweep, IdentificationErrorRate  # noqa: E402
from known_speakers_bench import make_clips  # noqa: E402
from sweep_bench import card, make_config, trials  # noqa: E402
from sweep_dataset_bench import SR, make_dataset  # noqa: E402

NAMES = ("alice", "bob", "carol", "dan")


def profiled(call, tags):
    """the CUDA-event milliseconds of ``tags`` over one call"""
    lib = _lib.lib()
    lib.dg_profile_report(ctypes.create_string_buffer(1 << 16), 1 << 16)     # drop earlier records
    lib.dg_profile_enable(1)
    try:
        call()
        buf = ctypes.create_string_buffer(1 << 16)
        lib.dg_profile_report(buf, len(buf))
    finally:
        lib.dg_profile_enable(0)
    report = json.loads(buf.value.decode())
    return {tag: report[tag]["ms"] for tag in tags if tag in report}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
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
    clips = make_clips(8)
    enrolled = enroll(config, clips)
    gallery = KnownSpeakers(NAMES, enrolled.centroids[:len(NAMES)])
    sweep = HyperParameterSweep(config)
    plain = DatasetSweep(config, files, sweep=sweep)
    seeded = DatasetSweep(config, files, sweep=sweep, speakers=gallery)
    result["dataset_chunks"] = plain.num_chunks
    result["seed_bytes_256"] = len(files) * 256 * len(NAMES) * seeded.emb.shape[-1] * 8
    cases = {"unseeded_der": (plain, None), "seeded_der": (seeded, None), "seeded_ier": (seeded, IdentificationErrorRate())}
    for ds, metric in cases.values():                                   # warm-up of the dataset-sized buffers
        ds.score(trials(4), metric)
    rows = {name: {} for name in cases}
    for _ in range(args.rounds):
        for T in (1, 16, 256):
            tr = trials(T)
            for name, (ds, metric) in cases.items():
                ds.score(tr, metric)
                s = ds.timing["score"]
                best = rows[name].get(T)
                rows[name][T] = s if best is None else min(best, s)
    result["score_device_s"] = rows
    tr = trials(256)
    result["profile_256_ms"] = {name: profiled(lambda: ds.score(tr, metric), ("sweep_seed", "der_score", "cluster_sweep"))
                                for name, (ds, metric) in cases.items()}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
