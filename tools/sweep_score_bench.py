"""Measures DER scoring of sweep trials (HyperParameterSweep.score, dg_sweep_score) on the GPU and prints one JSON line (and
writes it to --out if given).

Input: the seeded synthetic 30-minute file of tools/sweep_bench.py and a seeded synthetic 5-speaker reference with
overlapping speech.  For T in {16, 256, 1024} trials: the network pass (once per file), dg_sweep_score (CUDA events around
the synchronous call) and the host time of the whole score() call.  For T in {16, 256} also what scoring replaces: run()
(network pass, dg_sweep_run, Annotation assembly) plus oracle/der.py per trial on the host, and whether its components equal
the device's bit for bit.  The card's name and power limit are recorded with the numbers.

    python tools/sweep_score_bench.py [--minutes 30] [--out /tmp/sweep_score_bench.json]
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
from diart_b200.core import Annotation, Segment  # noqa: E402
from diart_b200.tune import HyperParameterSweep  # noqa: E402
from oracle.der import der_components  # noqa: E402
from sweep_bench import card, make_config, trials  # noqa: E402


def synth_reference(seed, n_speakers, duration):
    rng = np.random.default_rng(seed)
    ref, n = Annotation(uri="synth"), 0
    for k in range(n_speakers):
        t = rng.uniform(0.0, 5.0)
        while t < duration:
            length = rng.uniform(0.3, 9.0)
            ref[Segment(t, min(t + length, duration)), n] = f"spk{k}"
            n += 1
            t += length + rng.uniform(0.0, 12.0)
    return ref


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=30.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    result = {"card": card()}
    config = make_config(dev)
    x = synth.synth_audio(int(args.minutes * 60 * 16000), seed=2024, num_speakers=5)
    ref = synth_reference(2025, 5, len(x) / 16000)
    sweep = HyperParameterSweep(config)
    sweep.score(x, ref, trials(4))                          # warm-up: handles, pinned staging, first-use attributes
    result["file_seconds"] = len(x) / 16000
    rows = {}
    for T in (16, 256, 1024):
        best = None
        for _ in range(3):
            t0 = time.perf_counter()
            comp = sweep.score(x, ref, trials(T))
            host = time.perf_counter() - t0
            tm = dict(sweep.timing, host=host)
            best = tm if best is None else {k: min(best[k], v) for k, v in tm.items()}
        rows[T] = {"network_s": best["network"], "score_device_s": best["score"], "score_call_s": best["host"],
                   "best_der": float(comp.der.min())}
        if T in (16, 256):
            t0 = time.perf_counter()
            preds = sweep.run(x, uri="synth", trials=trials(T))
            t1 = time.perf_counter()
            want = np.stack([der_components(ref, p) for p in preds])
            t2 = time.perf_counter()
            rows[T].update({"replaced_run_s": t1 - t0, "replaced_oracle_der_s": t2 - t1,
                            "replaced_total_s": t2 - t0, "components_equal": bool(np.array_equal(comp.as_array(), want))})
    result["trials"] = rows
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    if not all(r["components_equal"] for r in rows.values() if "components_equal" in r):
        sys.exit("the device components differ from the host oracle")


if __name__ == "__main__":
    main()
